"""``matmul_fp8``: activation x group-quantised FP8 weight (reference ``ops/fp_quantizer/fp8_gemm.py:16``).

The weight arrives in :class:`FP_Quantize`'s flat layout (groups of ``quantization_group_size`` consecutive elements of
the row-major ``[K, N]`` tensor, one fp32 scale per group). It is expanded once by the dequantisation kernel and the
product runs on the library bf16 GEMM -- on H100 the expansion is bandwidth-trivial next to the GEMM for every ``M`` the
training path uses. (Serving-side weight-only GEMMs with their own ``[N, K]`` group layout and a fused wgmma kernel live in
``inference/quantization``.)"""
import torch


def matmul_fp8(inp, weight, scale, quantization_group_size, quantizer):
    assert quantizer.group_size == quantization_group_size, "quantizer was built for another group size"
    w = quantizer.dequantize(weight, scale=scale)
    if w.dim() != 2:
        w = w.view(quantizer.orig_shape)
    return torch.matmul(inp, w.to(inp.dtype))


matmul_fp8_fallback = matmul_fp8
