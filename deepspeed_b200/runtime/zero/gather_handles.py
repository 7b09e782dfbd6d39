"""Completion handles for parameter all-gathers and the int8 weight codec used by ZeRO++ quantised gathers
(reference ``runtime/zero/partition_parameters.py:603-830``: ``NoGatherHandle``, ``AllGatherHandle``,
``AllGatherCoalescedHandle``, ``MultipleAllGatherHandles``, ``AllReduceCoalescedHandle``, ``QuantizationInfo``,
``CUDAQuantizer``).

A handle owns (a) the communication work object(s) and (b) the rule that turns the gathered flat buffer back into
``param.data`` views.  ``wait()`` is idempotent; parameters flip INFLIGHT → AVAILABLE exactly once."""
import math
from typing import List, Optional

import torch


def _status():
    from .partition_parameters import ZeroParamStatus
    return ZeroParamStatus


def _require_inflight(param):
    if param.ds_status != _status().INFLIGHT:
        raise RuntimeError(f"expected param {param.ds_summary()} to be inflight")


class QuantizationInfo:
    """Side-band of a quantised gather: codec + the int8 payload / scale buffers and their work handles."""
    __slots__ = ("quantized_param", "backend", "quant_handle", "scale_buffer", "partition_sz", "world_size", "scale_handle")

    def __init__(self):
        for s in self.__slots__:
            setattr(self, s, None)


class CUDAQuantizer:
    """Symmetric int8 group codec backed by the native quantiser op.  Group count is chosen so that groups are a
    multiple of 8 elements, no larger than the kernel takes for the dtype (8192 16-bit or 4096 fp32 elements), and as
    close to ``target_group_size`` as divisibility allows (cached per tensor size and dtype)."""
    async_flag = True
    target_group_size = 8000
    group_size_cache = {}

    @staticmethod
    def max_group_size(dtype):
        """Largest group the quantize kernel accepts: one CTA keeps 4 16-byte vectors per thread in registers."""
        return 4096 if dtype == torch.float32 else 8192

    def _groups_for(self, n, dtype=torch.bfloat16):
        key = (n, self.max_group_size(dtype))
        g = self.group_size_cache.get(key)
        if g is not None:
            return g
        assert n % 8 == 0, f"quantised weights need a multiple of 8 elements, got {n}"
        units = n // 8  # groups must divide ``units``
        lo = max(1, math.ceil(n / key[1]))
        want = max(lo, math.ceil(n / self.target_group_size))
        cands = [d for d in _divisors(units) if d >= lo]
        assert cands and cands[0] < n, f"adaptive grouping cannot find a group size for a tensor of {n} elements"
        # largest group (fewest groups) that still respects the 8k target; else the smallest legal count
        below = [d for d in cands if d >= want]
        g = below[0] if below else cands[-1]
        self.group_size_cache[key] = g
        return g

    def quantize(self, param, groups=None):
        from deepspeed_b200.ops.quantizer import quantizer as Q
        groups = groups or self._groups_for(param.numel(), param.dtype)
        return Q.quantize(param.contiguous().view(-1), groups, 8, Q.Symmetric)

    def dequantize(self, quantized_param, scale, dtype=torch.bfloat16):
        from deepspeed_b200.ops.quantizer import quantizer as Q
        return Q.dequantize(quantized_param, scale, scale.numel(), 8, Q.Symmetric, dtype=dtype)


def _divisors(n):
    small, large = [], []
    i = 1
    while i * i <= n:
        if n % i == 0:
            small.append(i)
            if i != n // i:
                large.append(n // i)
        i += 1
    return small + large[::-1]


class NoGatherHandle:
    """World-size-1 fast path: the "gather" is a device move of the local slice."""

    def __init__(self, param):
        _require_inflight(param)
        piece = param.ds_tensor
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else piece.device
        param.data = piece.data.to(dev, non_blocking=True)[:param.ds_numel].view(param.ds_shape)
        self._param = param

    def wait(self, **kw):
        if self._param.data.is_cuda:
            torch.cuda.current_stream().synchronize()
        self._param.ds_status = _status().AVAILABLE


class NoGatherCoalescedHandle:

    def __init__(self, params: List):
        self._handles = [NoGatherHandle(p) for p in params]
        self._done = False

    def wait(self, **kw):
        if not self._done:
            for h in self._handles:
                h.wait()
            self._done = True


class AllGatherHandle:
    """One parameter, one collective.  ``flat`` is the gathered ``world × slice`` buffer the work object fills."""

    def __init__(self, handle, param, quantization: Optional[QuantizationInfo] = None, flat: Optional[torch.Tensor] = None):
        _require_inflight(param)
        self._work, self._param, self._q, self._flat = handle, param, quantization, flat

    def wait(self, handle_dependency=True):
        if self._work is not None:
            self._work.wait()
        p = self._param
        if self._q is not None:
            if self._q.quant_handle is not None:
                self._q.quant_handle.wait()
            full = self._q.backend.dequantize(self._q.quantized_param, self._q.scale_buffer, dtype=p.dtype)
            p.data = full.view(-1)[:p.ds_numel].view(p.ds_shape).to(p.ds_tensor.device if not torch.cuda.is_available()
                                                                     else full.device)
        elif self._flat is not None:
            p.data = self._flat[:p.ds_numel].view(p.ds_shape)
        p.ds_status = _status().AVAILABLE
        self._work = None


class AllGatherCoalescedHandle:
    """Several parameters gathered by ONE collective into a ``world × Σslice`` buffer: rank r's contribution holds its
    slice of every parameter back to back, so parameter i is re-assembled from ``world`` strided pieces."""
    data_buffer = []

    def __init__(self, allgather_handle, params: List, partitions: List[torch.Tensor], world_size: int,
                 use_secondary_tensor=False, quantization: Optional[QuantizationInfo] = None):
        for p in params:
            _require_inflight(p)
        self._work, self._params, self._parts, self._world = allgather_handle, params, partitions, world_size
        self._secondary, self._q, self._done = use_secondary_tensor, quantization, False

    def wait(self, handle_dependency=True):
        if self._done:
            return
        if self._work is not None:
            self._work.wait()
        parts = self._parts
        if self._q is not None:
            if self._q.quant_handle is not None:
                self._q.quant_handle.wait()
            flat = self._q.backend.dequantize(self._q.quantized_param, self._q.scale_buffer, dtype=self._params[0].dtype)
            sz = self._q.partition_sz
            parts = [flat.view(-1).narrow(0, r * sz, sz) for r in range(self._world)]
        off = 0
        for p in self._params:
            piece_attr = "ds_secondary_tensor" if self._secondary and getattr(p, "ds_secondary_tensor", None) is not None \
                else "ds_tensor"
            n = getattr(p, piece_attr).numel()
            full = torch.cat([parts[r].narrow(0, off, n) for r in range(self._world)]) if self._world > 1 \
                else parts[0].narrow(0, off, n)
            p.data = full[:p.ds_numel].view(p.ds_shape)
            p.ds_status = _status().AVAILABLE
            if handle_dependency and full.is_cuda:
                full.record_stream(torch.cuda.current_stream())
            off += n
        if not handle_dependency:
            AllGatherCoalescedHandle.data_buffer.append(parts)
        self._done = True

    @staticmethod
    def free_buffer():
        AllGatherCoalescedHandle.data_buffer = []


class MultipleAllGatherHandles:
    """Fan-in over several handles (one per dtype bucket)."""

    def __init__(self, handles: List):
        self.handles = list(handles)

    def wait(self, handle_dependency=True):
        for h in self.handles:
            h.wait(handle_dependency) if isinstance(h, (AllGatherHandle, AllGatherCoalescedHandle)) else h.wait()


class AllReduceCoalescedHandle:
    """Replicated-parameter path (``ds_tensor`` zero-padded everywhere except on the owner; a sum re-creates it)."""

    def __init__(self, handle, params: List):
        for p in params:
            _require_inflight(p)
        self._work, self._params, self._done = handle, params, False

    def wait(self, **kw):
        if self._done:
            return
        if self._work is not None:
            self._work.wait()
        for p in self._params:
            p.ds_status = _status().AVAILABLE
        self._done = True
