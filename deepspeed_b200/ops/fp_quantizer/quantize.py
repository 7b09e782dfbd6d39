"""Minifloat group quantizer: FP8 (E4M3 / E5M2), FP6 (E3M2), FP4 (E2M1), FP12 (E4M7).

Parity target: reference ``ops/fp_quantizer/quantize.py`` (``FP_Quantize``: ``quantize``, ``dequantize``,
``selective_dequantize``, ``get_scales``) over ``csrc/fp_quantizer/fp_quantize.cu`` (N6).
"""
import ctypes

import torch

from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.quantizer.quantizer import _to_grid

_MANTISSA = {8: 3, 6: 2, 4: 1, 12: 7}


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _fmt_max(bits, m):
    if bits == 8:
        return 448.0 if m == 3 else 57344.0
    e = bits - 1 - m
    bias = 2**(e - 1) - 1
    return (2 - 2.0**-m) * 2.0**((2**e - 1) - bias)


def _host_codec(v, bits, m):
    """Round ``v`` (already divided by the group scale) to the format's grid; returns float values."""
    if bits == 8:
        dt = torch.float8_e4m3fn if m == 3 else torch.float8_e5m2
        return v.clamp(-_fmt_max(bits, m), _fmt_max(bits, m)).to(dt).float()
    e = bits - 1 - m
    bias = 2**(e - 1) - 1
    a = v.abs().clamp(max=_fmt_max(bits, m))
    min_normal = 2.0**(1 - bias)
    sub_step = 2.0**(1 - bias - m)
    ex = torch.floor(torch.log2(a.clamp(min=1e-30)))
    step = torch.where(a < min_normal, torch.full_like(a, sub_step), 2.0**(ex - m))
    t = a / step
    q = (torch.floor(t) + (t - torch.floor(t) >= 0.5)) * step  # ties away; t + 0.5 could round up from below a tie
    return torch.sign(v) * q.clamp(max=_fmt_max(bits, m))


class Quantizer:

    def __init__(self, group_size=512):
        self.group_size = group_size


class FP_Quantize(Quantizer):

    def __init__(self, quantization_config=None, group_size=512):
        if quantization_config is not None:
            group_size = getattr(quantization_config, "group_size", group_size)
        super().__init__(group_size)
        self.orig_dtype = None
        self.orig_shape = None
        self.scales = None
        self.q_bits = 8
        self.q_mantisa_bits = 3

    def quantize(self, input, q_bits=8, q_mantisa_bits=3, stochastic_mode=False, return_meta_tensor=False):
        assert input.dtype in (torch.bfloat16, torch.float16, torch.float32)
        assert q_bits in _MANTISSA, f"unsupported q_bits {q_bits}"
        if q_bits != 8:
            q_mantisa_bits = _MANTISSA[q_bits]
        self.orig_dtype, self.orig_shape = input.dtype, input.shape
        self.q_bits, self.q_mantisa_bits = q_bits, q_mantisa_bits
        x = input.contiguous().reshape(-1)
        n = x.numel()
        gs = self.group_size
        if n % gs:  # a ragged tail is quantized as one zero-padded group (reference quantize.py: num_groups rounds up)
            x = torch.nn.functional.pad(x, (0, gs - n % gs))
        groups = x.numel() // gs
        bpg = (gs * q_bits + 7) // 8
        if x.is_cuda:
            q = torch.empty(groups * bpg, dtype=torch.uint8, device=x.device)
            scales = torch.empty(groups, dtype=torch.float32, device=x.device)
            seed = int(torch.randint(0, 2**31 - 1, (1, )).item()) if stochastic_mode else 0
            rc = N.cuda().dsb_fp_quantize(_p(x), _p(q), _p(scales), ctypes.c_int64(groups), gs, q_bits, q_mantisa_bits,
                                          N.dt(x), int(stochastic_mode), ctypes.c_uint32(seed), N.stream())
            N.check(rc, "fp_quantize")
        else:
            g = x.float().reshape(groups, gs)
            amax = g.abs().amax(1, keepdim=True)
            # the kernel's scale: NaN for a group holding a NaN or an inf, at least the smallest fp32 subnormal
            scales = torch.where(amax > 0, (amax / _fmt_max(q_bits, q_mantisa_bits)).clamp(min=2.0**-149),
                                 torch.ones_like(amax))
            scales = torch.where(torch.isfinite(amax), scales, float("nan")).reshape(groups)
            # host tier keeps decoded values (1 float per code) -- layout is an implementation detail
            q = _host_codec(_to_grid(g, scales[:, None]), q_bits, q_mantisa_bits).reshape(-1)
        self.scales = scales
        if return_meta_tensor:
            return q, scales
        return q

    def get_scales(self):
        return self.scales

    @property
    def scale(self):  # the reference keeps the group scales under this name
        return self.scales

    def to(self, *args, **kwargs):
        if self.scales is not None:
            self.scales = self.scales.to(*args, **kwargs)
        return self

    def dequantize(self, input_q, fp_out=None, q_bits=None, q_mantisa_bits=None, scale=None):
        q_bits = q_bits or self.q_bits
        m = q_mantisa_bits if q_mantisa_bits is not None else (self.q_mantisa_bits if q_bits == 8 else _MANTISSA[q_bits])
        scales = scale if scale is not None else self.scales
        gs = self.group_size
        groups = scales.numel()
        dtype = self.orig_dtype or torch.bfloat16
        want = self.orig_shape.numel() if self.orig_shape is not None else groups * gs
        padded = want < groups * gs  # the last group carries zero padding
        if input_q.is_cuda:
            direct = fp_out is not None and not padded
            out = fp_out if direct else torch.empty(groups * gs, dtype=dtype, device=input_q.device)
            rc = N.cuda().dsb_fp_dequantize(_p(input_q), _p(scales), _p(out), ctypes.c_int64(groups), gs, q_bits, m,
                                            N.dt(out), ctypes.c_void_p(0), 1, N.stream())
            N.check(rc, "fp_dequantize")
        else:
            out = (input_q.reshape(groups, gs) * scales[:, None]).to(dtype).reshape(-1)
            direct = False
        if padded:
            out = out[:want]
        if fp_out is not None and not direct:
            fp_out.copy_(out.view_as(fp_out))
            out = fp_out
        return out.view(self.orig_shape) if self.orig_shape is not None and out.numel() == self.orig_shape.numel() else out

    def selective_dequantize(self, input_q, indexes, fp_out=None, q_bits=None, q_mantisa_bits=None, scale=None):
        """Dequantize only rows ``indexes`` of the original (>= 2-D) tensor's leading dimension."""
        assert self.orig_shape is not None and len(self.orig_shape) >= 2
        q_bits = q_bits or self.q_bits
        m = q_mantisa_bits if q_mantisa_bits is not None else (self.q_mantisa_bits if q_bits == 8 else _MANTISSA[q_bits])
        scales = scale if scale is not None else self.scales
        gs = self.group_size
        row_elems = self.orig_shape.numel() // self.orig_shape[0]
        assert row_elems % gs == 0
        gpr = row_elems // gs
        idx = indexes.to(torch.int32).contiguous()
        out_groups = idx.numel() * gpr
        dtype = self.orig_dtype or torch.bfloat16
        if input_q.is_cuda:
            out = fp_out if fp_out is not None else torch.empty(out_groups * gs, dtype=dtype, device=input_q.device)
            rc = N.cuda().dsb_fp_dequantize(_p(input_q), _p(scales), _p(out), ctypes.c_int64(out_groups), gs, q_bits, m,
                                            N.dt(out), _p(idx), gpr, N.stream())
            N.check(rc, "fp_selective_dequantize")
        else:
            full = (input_q.reshape(-1, gs) * scales[:, None]).to(dtype).reshape(self.orig_shape[0], -1)
            out = full[indexes.long()].reshape(-1)
        return out.view(idx.numel(), *self.orig_shape[1:])
