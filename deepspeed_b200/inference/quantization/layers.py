"""Weight-only quantized linears for inference (reference ``inference/quantization/layers.py``,
``inference/v2/modules/implementations/linear/quantized_linear.py`` (FP6 ``wf6af16``), ``ops/fp_quantizer``).

Weights are stored group-quantised (int8/int4 via ``quant.cu`` or FP8/FP6 via ``fp_quantize``); at run time the
weight is dequantised tile-wise into bf16 and fed to the tensor-core GEMM.  For decode-sized inputs (few rows)
the op is bandwidth bound on the *weight* bytes, so 8-/6-bit storage is the win; the dequant kernel streams the
packed bytes once.
"""
import torch
import torch.nn.functional as F

from deepspeed_b200.ops.quantizer import quantizer as Q


class QuantizedWeight:
    """Packed weight + group params.  ``mode``: int8 | int4 | fp8 | fp6"""

    def __init__(self, q, params, shape, mode, group_size, dtype):
        self.q, self.params, self.shape, self.mode, self.group_size, self.dtype = q, params, tuple(shape), mode, group_size, dtype

    @property
    def is_cuda(self):
        return self.q.is_cuda

    def dequantize(self):
        n = self.shape[0] * self.shape[1]
        groups = n // self.group_size
        if self.mode in ("int8", "int4"):
            return Q.dequantize(self.q, self.params, groups, 8 if self.mode == "int8" else 4, Q.Symmetric,
                                dtype=self.dtype).view(self.shape)
        from deepspeed_b200.ops.fp_quantizer.quantize import FP_Quantize
        fq = FP_Quantize(group_size=self.group_size)
        fq.orig_shape, fq.orig_dtype = torch.Size(self.shape), self.dtype
        bits, man = (8, 3) if self.mode == "fp8" else (6, 2)
        return fq.dequantize(self.q, q_bits=bits, q_mantisa_bits=man, scale=self.params).view(self.shape).to(self.dtype)


def quantize_weight(w, mode="int8", group_size=128):
    n = w.numel()
    while n % group_size:
        group_size //= 2
    groups = n // group_size
    if mode in ("int8", "int4"):
        q, params = Q.quantize(w.contiguous(), groups, 8 if mode == "int8" else 4, Q.Symmetric)
        return QuantizedWeight(q, params, w.shape, mode, group_size, w.dtype)
    if mode in ("fp8", "fp6", "wf6af16"):
        from deepspeed_b200.ops.fp_quantizer.quantize import FP_Quantize
        fq = FP_Quantize(group_size=group_size)
        bits, man = (8, 3) if mode == "fp8" else (6, 2)
        q, scale = fq.quantize(w.contiguous(), q_bits=bits, q_mantisa_bits=man, return_meta_tensor=True)
        return QuantizedWeight(q, scale, w.shape, "fp8" if mode == "fp8" else "fp6", group_size, w.dtype)
    raise ValueError(f"unknown quantization mode {mode}")


def maybe_quantized_linear(x, w, b=None):
    if isinstance(w, QuantizedWeight):
        y = _wq_gemv(x, w, b)
        if y is None:
            y = wq_tc_linear(x, w, b)
        if y is not None:
            return y
        w = w.dequantize()
    return F.linear(x, w, b)


_TC_MODES = {"int8": 0, "int4": 1, "fp8": 2, "fp6": 3}
# Row count up to which the fused kernel beats dequantise-once + bf16 GEMM, per weight format, measured on an H100 80GB HBM3
# at a 400 W power limit at [rows x 14336 x 4096] (scripts/bench_wq_tc.py), fused speedup at 128 / 256 / 512 / 1024 rows:
# int8 2.22x / 1.28x / 0.81x / 0.63x; int4 2.47x / 1.57x / 1.03x / 0.80x; fp8 2.69x / 1.65x / 1.02x / 0.78x;
# fp6 2.73x / 1.69x / 1.02x / 0.74x.  The kernel covers 128 tokens per CTA, so every further 128 rows re-read the weights.
WQ_TC_MAX_ROWS_BY_MODE = {"int8": 256, "int4": 512, "fp8": 512, "fp6": 512}
WQ_TC_MAX_ROWS = 512


def wq_tc_linear(x, qw: "QuantizedWeight", b=None, max_rows=None):
    """32 < rows <= ``WQ_TC_MAX_ROWS``: fused dequantise-in-shared-memory + wgmma GEMM (``csrc/cuda/wq_tc_gemm.cu``) for
    FP6 / FP8 / INT8 / INT4 weights -- the dequantised weight never exists in HBM.  None -> not eligible."""
    if not (x.is_cuda and x.dtype == torch.bfloat16 and qw.mode in _TC_MODES and qw.dtype == torch.bfloat16):
        return None
    x2 = x.reshape(-1, x.shape[-1])
    M, K = x2.shape
    N = qw.shape[0]
    limit = min(WQ_TC_MAX_ROWS, WQ_TC_MAX_ROWS_BY_MODE.get(qw.mode, WQ_TC_MAX_ROWS)) if max_rows is None else max_rows
    if M > limit or K != qw.shape[1] or K % 64 or qw.group_size % 64 or K % qw.group_size:
        return None
    from deepspeed_b200.ops import native as NV
    if x2.stride(1) != 1 or x2.stride(0) % 8 or x2.data_ptr() % 16:
        x2 = x2.contiguous()
    out = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
    bias = b.to(torch.bfloat16).contiguous() if b is not None else None
    rc = NV.cuda().dsb_wq_tc_gemm(NV.ptr(x2), NV.ptr(qw.q), NV.ptr(qw.params), NV.ptr(bias), NV.ptr(out), M, N, K,
                                  _TC_MODES[qw.mode], qw.group_size, x2.stride(0), out.stride(0), NV.stream())
    if rc == -3:
        return None
    NV.check(rc, "wq_tc_gemm")
    return out.view(*x.shape[:-1], N)


def _wq_gemv(x, qw: "QuantizedWeight", b):
    """Decode-sized inputs: fused in-register dequantisation + GEMV (``csrc/cuda/wq_gemm.cu``); None -> not eligible."""
    import ctypes
    if not (x.is_cuda and qw.mode in ("int8", "int4", "fp8") and x.dtype in (torch.bfloat16, torch.float16)):
        return None
    x2 = x.reshape(-1, x.shape[-1])
    M, K = x2.shape
    N = qw.shape[0]
    if M > 32 or K != qw.shape[1]:
        return None
    from deepspeed_b200.ops import native as NV
    x2 = x2.contiguous()
    out = torch.empty(M, N, dtype=x.dtype, device=x.device)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    bias = b.to(x.dtype).contiguous() if b is not None else None
    if qw.mode == "fp8":
        rc = NV.cuda().dsb_wq_gemv_fp8(p(x2), p(qw.q), p(qw.params), p(bias), p(out), M, N, K, qw.group_size, NV.dt(x2), NV.stream())
    else:
        rc = NV.cuda().dsb_wq_gemv(p(x2), p(qw.q), p(qw.params), p(bias), p(out), M, N, K, 8 if qw.mode == "int8" else 4,
                                   qw.group_size, NV.dt(x2), NV.stream())
    if rc == -3:
        return None
    NV.check(rc, "wq_gemv")
    return out.view(*x.shape[:-1], N)


class QuantizedLinear(torch.nn.Module):
    """Drop-in for nn.Linear holding a QuantizedWeight (reference ``QuantizedLinear``)."""

    def __init__(self, linear: torch.nn.Linear, mode="int8", group_size=128):
        super().__init__()
        self.qw = quantize_weight(linear.weight.data, mode, group_size)
        self.bias = linear.bias
        self.in_features, self.out_features = linear.in_features, linear.out_features

    def forward(self, x):
        return maybe_quantized_linear(x, self.qw, self.bias)


# ---- ZeRO-Inference style post-init quantisation wrappers (reference ``inference/quantization/layers.py:20-110``) ------
# One compat blob per ORIGINAL weight object: tied weights (embedding ↔ lm_head) are quantised once and shared.
quantized_weight_registry = {}
is_zero3_enabled = False


def get_quantize_weight_fn(quantizer, pre_quant_weight):
    """Deferred ``quantizer.quantize(weight)`` → ``(codes, scale, min)``."""

    def func():
        return quantizer.quantize(pre_quant_weight.data)

    return func


def get_quantized_weight_wrapper(model, pre_quant_weight, quantize_weight_fn):
    """The packed quantised parameter standing for ``pre_quant_weight`` (created on first request, then shared)."""
    from .utils import concat_to_compat_param
    key = id(pre_quant_weight)
    blob = quantized_weight_registry.get(key)
    if blob is None:
        codes, scale, mn = quantize_weight_fn()
        blob = concat_to_compat_param(codes, scale, mn)
        blob.quant_shape, blob.quant_groups = tuple(codes.shape), scale.numel()
        blob.quant_scale_shape, blob.quant_dtype = tuple(scale.shape), scale.dtype
        quantized_weight_registry[key] = blob
    elif is_zero3_enabled:
        from deepspeed_b200.runtime.zero import register_external_parameter
        register_external_parameter(model, blob)
    return blob


class QuantizedEmbedding(torch.nn.Embedding):
    """``nn.Embedding`` whose table is stored group-quantised (4 / 8 bit asymmetric); only the looked-up rows are
    dequantised when rows are whole groups, otherwise the table is dequantised transiently."""

    def __init__(self, config, pre_quant_layer: torch.nn.Embedding) -> None:
        from .utils import DeQuantizer, Quantizer
        w = pre_quant_layer.weight
        assert pre_quant_layer.max_norm is None and pre_quant_layer.norm_type == 2, "Not supported"
        assert not pre_quant_layer.scale_grad_by_freq and not pre_quant_layer.sparse, "Not supported"
        super().__init__(pre_quant_layer.num_embeddings, pre_quant_layer.embedding_dim, padding_idx=pre_quant_layer.padding_idx,
                         _weight=w, device=w.device, dtype=w.dtype)
        self.config = config
        self.weight = get_quantized_weight_wrapper(self, w, get_quantize_weight_fn(Quantizer(config), w))
        self.weight.dequantizer = DeQuantizer(config, w.dtype)

    def _table(self):
        from .utils import split_compat_param
        p = self.weight
        codes, scale, mn = split_compat_param(p.data, p.quant_shape, p.quant_groups, p.quant_dtype)
        return p.dequantizer.dequantize(codes, scale.view(p.quant_scale_shape), mn.view(p.quant_scale_shape))

    def forward(self, input):
        return torch.nn.functional.embedding(input, self._table(), self.padding_idx)
