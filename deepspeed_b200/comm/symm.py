"""Symmetric (peer-mapped) memory + in-kernel NVLink collectives.

This is the H100-native replacement for "NCCL call on a side stream" on the two ZeRO hot paths
(SURVEY.md 5.8): buffers are allocated with the CUDA VMM API, exported as POSIX file descriptors,
exchanged between the ranks of one node over a unix-domain socket (``SCM_RIGHTS``) and mapped into
every rank's address space, so a kernel can ``ld``/``st`` a peer's buffer over NVLink.  A
multicast object (NVLS) is bound on top when the driver supports it so ``multimem.ld_reduce`` /
``multimem.st`` can reduce / broadcast inside the NVSwitch.

Native parts: ``csrc/cuda/symm_mem.cpp`` (allocation, handle exchange, mapping) and
``csrc/cuda/symm_coll.cu`` (all-gather, reduce-scatter fused with scale + accumulate / Adam,
one-shot all-reduce, device barrier).  This module is the Python face.  The implementation is
filled in by ``_SymmContext``; when the arena cannot be created (single GPU, host tier, P2P
unavailable) every query returns ``None``/``False`` and callers use the NCCL path.
"""
import os
from typing import Dict, Optional

import torch

from deepspeed_b200.utils.logging import logger

_contexts: Dict[int, object] = {}
_disabled_reason: Optional[str] = None


def _env_enabled(explicit: bool) -> bool:
    v = os.environ.get("DSB200_SYMM", "")
    if v == "0":
        return False
    if v == "1":
        return True
    return explicit or os.environ.get("DSB200_SYMM_AUTO", "1") == "1"


def is_supported(group=None, explicit=False) -> bool:
    """True when a symmetric arena can be (or has been) created for ``group``."""
    global _disabled_reason
    if not torch.cuda.is_available() or not _env_enabled(explicit):
        return False
    if _disabled_reason is not None:
        return False
    try:
        from .symm_impl import probe
        ok, why = probe(group)
        if not ok:
            _disabled_reason = why
            logger.info(f"symmetric memory disabled: {why}")
        return ok
    except Exception as e:  # pragma: no cover - depends on the box
        _disabled_reason = repr(e)
        logger.warning(f"symmetric memory probe failed: {e!r}")
        return False


def get_context(group=None):
    key = id(group) if group is not None else 0
    if key in _contexts:
        return _contexts[key]
    if not is_supported(group, explicit=True):
        return None
    from .symm_impl import SymmContext
    try:
        ctx = SymmContext(group)
    except Exception as e:  # pragma: no cover
        global _disabled_reason
        _disabled_reason = repr(e)
        logger.warning(f"symmetric memory setup failed, using NCCL: {e!r}")
        return None
    _contexts[key] = ctx
    return ctx


def maybe_alloc(numel, dtype, device, group=None):
    """Allocate ``numel`` elements from the symmetric arena or return ``None``."""
    ctx = get_context(group)
    if ctx is None:
        return None
    return ctx.alloc(numel, dtype)


def try_one_shot_all_reduce(tensor, group=None) -> bool:
    ctx = _contexts.get(id(group) if group is not None else 0)
    if ctx is None or not ctx.owns(tensor):
        return False
    return ctx.all_reduce_(tensor)


def shutdown():
    for c in list(_contexts.values()):
        try:
            c.close()
        except Exception:
            pass
    _contexts.clear()
