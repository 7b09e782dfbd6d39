"""``out = hidden @ W^T`` through the autotuned GEMM (cuBLAS or the wgmma kernels).

Reference ``inference/v2/kernels/core_ops/blas_kernels/blas_linear.py``."""
import torch

from deepspeed_b200.ops import gemm

from ...ds_kernel import DSKernelBase, check_dtype


class BlasLibLinear(DSKernelBase):
    supported_dtypes = [torch.float16, torch.bfloat16, torch.float32]

    def __init__(self, fp_dtype):
        check_dtype(fp_dtype, "BlasLibLinear")
        self.dtype = fp_dtype

    def __call__(self, output: torch.Tensor, hidden_states: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
        x = hidden_states.reshape(-1, hidden_states.shape[-1])
        res = gemm.matmul_nt(x, weights) if x.is_cuda else torch.nn.functional.linear(x, weights)
        output.view(-1, output.shape[-1]).copy_(res)
        return output
