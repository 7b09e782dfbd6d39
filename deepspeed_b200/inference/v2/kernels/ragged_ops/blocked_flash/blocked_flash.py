"""Attention of a ragged batch over the blocked (paged) KV cache: every query token attends to keys ``[0, pos]`` of its sequence; GQA-shared split-KV kernel at decode sizes.

Reference ``inference/v2/kernels/ragged_ops/blocked_flash/blocked_flash.py``."""
import torch

from deepspeed_b200.ops.kernels import ragged_ops as R

from ...ds_kernel import DSKernelBase, check_dtype


class BlockedFlashAttn(DSKernelBase):
    supported_dtypes = [torch.float16, torch.bfloat16]

    def __init__(self, head_size: int, dtype) -> None:
        check_dtype(dtype, "BlockedFlashAttn")
        if head_size % 16 != 0:
            raise ValueError("Head size must be divisible by 16")
        self.head_size = head_size

    def __call__(self, out, qkv, kv_cache, seq_of, pos_of, block_table, n_q_heads, n_kv_heads, block_size, softmax_scale=None):
        """``qkv`` [T, (hq + 2 hkv) d] (K/V already appended to ``kv_cache`` by the rotary kernel)."""
        out.copy_(R.paged_attention(qkv, kv_cache, seq_of, pos_of, block_table, n_q_heads, n_kv_heads, self.head_size, block_size,
                                    softmax_scale))
        return out


def get_q_block_size(head_size: int) -> int:
    """Query tile of the prefill attention kernel: 128 rows (one wgmma M=128 tile) for every head size it supports."""
    if head_size % 16 != 0 or head_size > 256:
        raise ValueError(f"unsupported head size {head_size}")
    return 128


def get_kv_block_size(head_size: int) -> int:
    """Preferred KV-cache page: 128 tokens up to head size 128 (one TMA box per page), 64 above so a K+V page pair stays
    within the shared-memory stage budget."""
    if head_size % 16 != 0 or head_size > 256:
        raise ValueError(f"unsupported head size {head_size}")
    return 128 if head_size <= 128 else 64
