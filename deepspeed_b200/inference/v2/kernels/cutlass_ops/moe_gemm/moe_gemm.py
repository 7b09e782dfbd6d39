"""Grouped GEMM over expert-sorted rows.

Reference ``inference/v2/kernels/cutlass_ops/moe_gemm/moe_gemm.py``."""
import torch

from deepspeed_b200.utils.types import ActivationFuncType

from ...ds_kernel import DSKernelBase, check_dtype


class MoEGEMM(DSKernelBase):
    supported_dtypes = [torch.float16, torch.bfloat16, torch.float32]
    supported_act_fns = [ActivationFuncType.UNKNOWN, ActivationFuncType.GELU, ActivationFuncType.ReLU]

    def __init__(self, fp_dtype, act_fn=ActivationFuncType.UNKNOWN) -> None:
        check_dtype(fp_dtype, "MoEGEMM")
        if act_fn not in self.supported_act_fns:
            raise ValueError(f"Unsupported activation {act_fn}")
        self.act_fn = act_fn

    def __call__(self, ordered_output, ordered_input, weights, cumsum_rows, biases=None) -> None:
        """``weights`` [E, out, in]; expert e owns rows ``cumsum_rows[e-1]:cumsum_rows[e]`` of the sorted input."""
        from ... import moe_gemm
        if torch.is_tensor(cumsum_rows) and cumsum_rows.is_cuda and biases is None and torch.is_tensor(weights):
            # device-resident offsets -> single grouped wgmma launch, no host synchronisation
            off = torch.cat([cumsum_rows.new_zeros(1), cumsum_rows]).to(torch.int32)
            moe_gemm(ordered_input, weights, off, out=ordered_output)
            if self.act_fn == ActivationFuncType.GELU:
                ordered_output.copy_(torch.nn.functional.gelu(ordered_output))
            elif self.act_fn == ActivationFuncType.ReLU:
                ordered_output.relu_()
            return ordered_output
        ends = cumsum_rows.tolist() if torch.is_tensor(cumsum_rows) else list(cumsum_rows)
        offsets = [0] + [int(e) for e in ends]
        moe_gemm(ordered_input, weights, offsets, out=ordered_output)
        if biases is not None:
            for e in range(len(ends)):
                ordered_output[offsets[e]:offsets[e + 1]] += biases[e]
        if self.act_fn == ActivationFuncType.GELU:
            ordered_output.copy_(torch.nn.functional.gelu(ordered_output))
        elif self.act_fn == ActivationFuncType.ReLU:
            ordered_output.relu_()
        return ordered_output
