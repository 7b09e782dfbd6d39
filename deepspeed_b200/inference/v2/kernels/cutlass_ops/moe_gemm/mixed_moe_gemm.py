"""Grouped GEMM with weight-only-quantised expert weights.

Reference ``inference/v2/kernels/cutlass_ops/moe_gemm/mixed_moe_gemm.py`` (cutlass ``moe_gemm`` with a dequantising
prologue).  Here: ONE launch of the grouped form of the wgmma dequantise-in-shared-memory kernel
(``csrc/cuda/wq_tc_gemm.cu``): blockIdx.z = expert, the expert extents are read from the device-resident cumulative row
counts (no ``.tolist()`` host synchronisation, CUDA-graph capturable), the packed weights of all experts are stacked once."""
import torch

from deepspeed_b200.inference.quantization.layers import _TC_MODES, maybe_quantized_linear
from deepspeed_b200.utils.types import ActivationFuncType

from ...ds_kernel import DSKernelBase, check_dtype


class MixedMoEGEMM(DSKernelBase):

    def __init__(self, fp_dtype, act_fn=ActivationFuncType.UNKNOWN, num_bits: int = 8) -> None:
        check_dtype(fp_dtype, "MixedMoEGEMM", allow_fp32=False)
        if num_bits not in (4, 8):
            raise ValueError("num_bits must be 4 or 8")
        self.act_fn, self.num_bits = act_fn, num_bits
        self._stack = None  # (key, q [E, ...], params [E, ...], bias [E, N] | None)

    def _stacked(self, weights, biases):
        key = (tuple(id(w) for w in weights), None if biases is None else id(biases))
        if self._stack is None or self._stack[0] != key:
            q = torch.stack([w.q.reshape(-1) for w in weights]).contiguous()
            prm = torch.stack([w.params.reshape(-1).float() for w in weights]).contiguous()
            b = None
            if biases is not None:
                b = (torch.stack(list(biases)) if not torch.is_tensor(biases) else biases).to(torch.bfloat16).contiguous()
            self._stack = (key, q, prm, b)
        return self._stack[1:]

    def __call__(self, ordered_output, ordered_input, weights, scales, cumsum_rows, biases=None) -> None:
        """``weights``: list of QuantizedWeight, one per expert; ``cumsum_rows``: inclusive cumulative row counts [E]."""
        w0 = weights[0]
        x = ordered_input
        fused = (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_tensor(cumsum_rows) and cumsum_rows.is_cuda
                 and w0.mode in _TC_MODES and all(w.mode == w0.mode and w.shape == w0.shape for w in weights)
                 and x.shape[-1] % 64 == 0 and w0.group_size % 64 == 0 and x.shape[-1] % w0.group_size == 0
                 and x.stride(-1) == 1 and x.stride(0) % 8 == 0 and ordered_output.dtype == torch.bfloat16)
        if fused:
            from deepspeed_b200.ops import native as NV
            E, (N, K) = len(weights), w0.shape
            q, prm, b = self._stacked(weights, biases)
            offs = torch.zeros(E + 1, dtype=torch.int32, device=x.device)
            offs[1:] = cumsum_rows.to(torch.int32)
            rc = NV.cuda().dsb_wq_tc_gemm_grouped(NV.ptr(x), NV.ptr(q), NV.ptr(prm), NV.ptr(b), NV.ptr(ordered_output),
                                                  NV.ptr(offs), E, x.shape[0], N, K, _TC_MODES[w0.mode], w0.group_size,
                                                  x.stride(0), ordered_output.stride(0), NV.stream())
            if rc != -3:
                NV.check(rc, "wq_tc_gemm_grouped")
                return ordered_output
        ends = cumsum_rows.tolist() if torch.is_tensor(cumsum_rows) else list(cumsum_rows)  # host / unsupported layouts
        s = 0
        for e, t in enumerate(ends):
            t = int(t)
            if t > s:
                ordered_output[s:t] = maybe_quantized_linear(ordered_input[s:t], weights[e], None if biases is None else biases[e])
            s = t
        return ordered_output
