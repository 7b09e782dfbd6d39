"""Kernel namespace of the ragged engine (reference ``inference/v2/kernels/{core_ops,ragged_ops,cutlass_ops}``).
All device code lives in ``libdsb200_cuda.so``; this module re-exports the Python faces under the names the
reference's module layer uses."""
from deepspeed_b200.ops.kernels.ragged_ops import (kv_rotary_append as linear_blocked_kv_rotary,  # noqa: F401
                                                   paged_attention as blocked_flash, ragged_embed, row_gather as
                                                   logits_gather)
from deepspeed_b200.ops.kernels.moe_ops import top_k_gating, scatter as moe_scatter, gather as moe_gather  # noqa: F401
from deepspeed_b200.ops.kernels.transformer_ops import (rms_norm, layer_norm, gated_act as gated_activation,  # noqa: F401
                                                        bias_act as bias_activation)
from deepspeed_b200.ops.gemm import matmul_nt as blas_linear  # noqa: F401


def mixed_gemm(x, qweight, bias=None):
    """Weight-only-quantised GEMM (reference cutlass ``mixed_gemm``): ``qweight`` is a ``QuantizedWeight`` (int8/int4/fp8/fp6);
    it is dequantised group-wise into bf16 and multiplied on the tensor cores."""
    from deepspeed_b200.inference.quantization.layers import maybe_quantized_linear
    return maybe_quantized_linear(x, qweight, bias)


def moe_gemm(x_sorted, expert_weights, offsets, out=None):
    """Grouped GEMM over expert-sorted rows (reference cutlass ``moe_gemm``): ``x_sorted`` [rows, K] with expert e owning
    rows ``offsets[e]:offsets[e+1]``, ``expert_weights`` [E, N, K] (or a list).  On the device with bf16 stacked weights
    this is ONE persistent wgmma launch driven by the device-resident offsets (``gemm_grouped_nt_kernel``); otherwise
    one GEMM per non-empty expert."""
    import torch
    from deepspeed_b200.ops.kernels import gemm_sm100
    if torch.is_tensor(offsets) and gemm_sm100.supports_grouped(x_sorted, expert_weights, offsets.to(torch.int32)
                                                                if offsets.dtype != torch.int32 else offsets):
        return gemm_sm100.grouped_matmul_nt(x_sorted, expert_weights, offsets if offsets.dtype == torch.int32 else
                                            offsets.to(torch.int32), out=out)
    off = offsets.tolist() if torch.is_tensor(offsets) else list(offsets)
    E = len(off) - 1
    n_out = expert_weights[0].shape[0]
    if out is None:
        out = torch.empty(x_sorted.shape[0], n_out, dtype=x_sorted.dtype, device=x_sorted.device)
    for e in range(E):
        s, t = off[e], off[e + 1]
        if t > s:
            torch.mm(x_sorted[s:t], expert_weights[e].t(), out=out[s:t])
    return out
