"""Base of the v1 inference op bindings (reference ``ops/transformer/inference/op_binding/base.py``).

The reference resolves each op to a ``*_fp16`` / ``*_bf16`` / ``*_fp32`` symbol of one monolithic extension.  Here every
op is a thin callable over the typed sm_90a kernels in ``ops/kernels`` (dtype dispatch happens in the C ABI), with a
torch path for host tensors, so a binding holds nothing but the layer config.
"""
import torch

from ..config import DeepSpeedInferenceConfig


class BaseOp(torch.nn.Module):

    def __init__(self, config: DeepSpeedInferenceConfig = None):
        super().__init__()
        self.config = config if config is not None else DeepSpeedInferenceConfig()

    @property
    def eps(self):
        return getattr(self.config, "epsilon", 1e-5)


def gemm_linear(x, weight, bias=None):
    """``x @ weight^T (+ bias)`` for the inference op bindings: bf16 CUDA problems with at least one 256x128 tile go to the
    framework's wgmma GEMM through :mod:`deepspeed_b200.ops.gemm` (persisted per-shape choice vs cuBLAS), weight-only
    quantised weights to the fused dequant kernels, everything else (decode-sized rows, fp16/fp32, host) to the library --
    the role of the reference's ``cublas_gemm_ex`` calls in ``csrc/transformer/inference/csrc/pt_binding.cpp``."""
    import torch.nn.functional as F
    from deepspeed_b200.inference.quantization.layers import QuantizedWeight, maybe_quantized_linear
    if isinstance(weight, QuantizedWeight):
        return maybe_quantized_linear(x, weight, bias)
    if x.is_cuda and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and weight.dim() == 2:
        x2 = x.reshape(-1, x.shape[-1])
        if x2.shape[0] >= 256 and x2.is_contiguous() and weight.is_contiguous():
            from deepspeed_b200.ops import gemm
            y = gemm.matmul_nt(x2, weight)
            if bias is not None:
                y = y + bias
            return y.view(*x.shape[:-1], weight.shape[0])
    return F.linear(x, weight, bias)
