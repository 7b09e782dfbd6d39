"""Group-wise integer quantization ops (python face of ``csrc/cuda/quant.cu``).

Parity target: reference ``ops/quantizer/quantizer.py`` + ``csrc/quantization/pt_binding.cpp:372-401``
(``quantize``, ``dequantize``, ``swizzle_quant``, ``quantized_reduction``, ``loco_*``, ``ds_quantize_*``,
``ds_sr_quantize_*``).  CUDA tensors use the sm_90a kernels; host tensors use an equivalent torch path so
ZeRO++ logic is testable on CPU.
"""
import ctypes

import torch

from deepspeed_b200.ops import native as N

Symmetric, Asymmetric = 0, 1


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _fma32(a, b, c):
    """fp32 ``a * b + c`` rounded once, like the kernels' ``__fmaf_rn``.  The float64 product of two fp32 values is
    exact, but the float64 sum may round; rounding that sum to fp32 again is only wrong when it lands exactly on an fp32
    midpoint, and then the sum's exact error (TwoSum) says which neighbour the exact value is nearer to."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.float()
    d = s - r.double()
    up, dn = torch.nextafter(r, torch.full_like(r, float("inf"))), torch.nextafter(r, torch.full_like(r, -float("inf")))
    r = torch.where((err > 0) & (d > 0) & (d == (up.double() - r.double()) / 2), up, r)
    return torch.where((err < 0) & (d < 0) & (-d == (r.double() - dn.double()) / 2), dn, r)


def _to_grid(x, scale):
    """``x / scale`` as the kernels compute it: times the fp32 reciprocal, or divided when that overflows."""
    inv = 1.0 / scale
    return torch.where(torch.isfinite(inv), x * inv, x / scale)


def _host_codes(g, bits, sym, stochastic=False):
    """Codes (as floats) of the groups in the rows of fp32 ``g``, with the kernels' arithmetic: the scale is the
    group's range over ``2^bits`` steps (at least the smallest fp32 subnormal), ``x * (1/scale)`` through the fp32
    reciprocal (a division when that overflows), round half to even, clamp.  A group whose range is not finite (it
    holds a NaN or an inf, or its asymmetric range overflows) gets a NaN scale and the lowest code everywhere, so all of
    it dequantizes to NaN.  Returns ``(v, scale, offset)``."""
    nan = torch.full_like(g[:, :1], float("nan"))
    if sym:
        span, offset = g.abs().amax(dim=1, keepdim=True), torch.zeros_like(nan)
        lo_q, hi_q, steps = -2**(bits - 1), 2**(bits - 1) - 1, 2**(bits - 1)  # amax -> 2^(b-1); +side saturates
    else:
        offset = g.amin(dim=1, keepdim=True)
        span = g.amax(dim=1, keepdim=True) - offset
        lo_q, hi_q, steps = 0, 2**bits - 1, 2**bits
    bad = ~torch.isfinite(span)
    scale = torch.where(bad, nan, torch.where(span > 0, (span / steps).clamp(min=2.0**-149), torch.ones_like(span)))
    v = _to_grid(g - offset, scale)
    if stochastic:  # floor(v + r), exactly
        fl = torch.floor(v)
        v = fl + (v - fl >= 1.0 - torch.rand_like(v))
    else:
        v = torch.round(v)
    v = torch.where(bad, torch.full_like(v, lo_q), v.clamp(lo_q, hi_q))
    return v, scale, offset


def _host_quant(x, groups, bits, sym, stochastic=False):
    return _host_pack(*_host_codes(x.reshape(groups, -1).float(), bits, sym, stochastic), bits, sym)


def _host_pack(v, scale, offset, bits, sym):
    groups = v.shape[0]
    q = v.to(torch.int32)
    params = scale.reshape(groups) if sym else torch.cat([scale, offset], dim=1)
    if bits == 8:
        out = (q if sym else q - 128).to(torch.int8)
    else:
        qq = q & 0xf
        out = (qq[:, 0::2] | (qq[:, 1::2] << 4)).to(torch.uint8).view(torch.int8)
    return out, params.float()


def _host_dequant(q, params, groups, bits, sym, dtype):
    q = q.reshape(groups, -1)
    if bits == 8:
        v = q.to(torch.int32) if sym else q.to(torch.int32) + 128
    else:
        b = q.view(torch.uint8).to(torch.int32)
        lo, hi = b & 0xf, b >> 4
        v = torch.stack([lo, hi], dim=2).reshape(groups, -1)
        if sym:
            v = torch.where(v >= 8, v - 16, v)
    if sym:
        return (v.float() * params.reshape(groups, 1)).to(dtype)
    p = params.reshape(groups, 2)
    return _fma32(v.float(), p[:, :1], p[:, 1:]).to(dtype)


def aligned_group_size(n, target=2048):
    """Group size for quantising ``n`` elements that the device kernels accept (a multiple of 8, at most ``target``);
    callers pad ``n`` up to a multiple of it."""
    return target if n >= target else max(8, (n + 7) // 8 * 8)


def quantize(x, groups, num_bits=8, q_type=Symmetric, group_perm=None, stochastic=False, seed=0):
    """Returns ``(q, params)``: ``q`` int8 (two values per byte for 4 bit), ``params`` fp32 ``[groups]``
    (symmetric: scale) or ``[groups, 2]`` (asymmetric: scale, offset)."""
    x = x.contiguous()
    n = x.numel()
    assert n % groups == 0
    gs = n // groups
    sym = q_type == Symmetric
    if x.dim() > 1 and (num_bits == 8 or x.shape[-1] % 2 == 0):
        # shaped in -> shaped out (the reference binding keeps the activation's shape; 4 bit halves the last dim)
        q, params = quantize(x.view(-1), groups, num_bits, q_type, group_perm, stochastic, seed)
        return q.view(*x.shape[:-1], x.shape[-1] if num_bits == 8 else x.shape[-1] // 2), params
    if not x.is_cuda:
        q, params = _host_quant(x, groups, num_bits, sym, stochastic)
        if group_perm is not None:
            inv = torch.empty_like(group_perm)
            q2, p2 = torch.empty_like(q), torch.empty_like(params)
            q2[group_perm.long()] = q
            p2[group_perm.long()] = params
            q, params = q2, p2
        return q.reshape(-1), params
    q = torch.empty(n if num_bits == 8 else n // 2, dtype=torch.int8, device=x.device)
    params = torch.empty(groups if sym else groups * 2, dtype=torch.float32, device=x.device)
    rc = N.cuda().dsb_quantize(_p(x), _p(q), _p(params), ctypes.c_int64(groups), gs, num_bits, int(sym), N.dt(x),
                               _p(group_perm), int(stochastic), ctypes.c_uint32(seed & 0xffffffff), N.stream())
    N.check(rc, "quantize")
    return q, (params if sym else params.view(groups, 2))


def loco_quantize(x, err, groups, num_bits=4, beta=0.8, reset=False):
    """LoCo error-feedback quantisation in one pass: ``q = Q(x + err)`` (symmetric, ``groups`` groups) and
    ``err <- beta * err + (1 - beta) * ((x + err) - deQ(q))`` in place (``err`` fp32, same numel; zeroed when ``reset``).
    Returns ``(q, params)`` like :func:`quantize` (reference ``loco_swizzled_quant``, ``csrc/quantization/swizzled_quantize.cu``)."""
    x = x.contiguous()
    n = x.numel()
    assert n % groups == 0 and err.numel() == n and err.dtype == torch.float32 and err.is_contiguous()
    gs = n // groups
    if not x.is_cuda:
        comp = x.reshape(groups, -1).float() + err.reshape(groups, -1)
        v, scale, offset = _host_codes(comp, num_bits, True)
        q, params = _host_pack(v, scale, offset, num_bits, True)
        ok = torch.isfinite(scale)  # a non-finite group leaves its error slice as it was
        e = err.view(groups, -1)
        if reset:
            new = torch.zeros_like(e)
        else:
            f = torch.tensor(beta, dtype=torch.float32)
            new = _fma32(f, e, (1.0 - f) * _fma32(-v, scale, comp))
        e.copy_(torch.where(ok, new, e))
        return q.reshape(-1), params
    q = torch.empty(n if num_bits == 8 else n // 2, dtype=torch.int8, device=x.device)
    params = torch.empty(groups, dtype=torch.float32, device=x.device)
    rc = N.cuda().dsb_loco_quantize(_p(x), _p(err), _p(q), _p(params), ctypes.c_int64(groups), gs, num_bits, N.dt(x),
                                    ctypes.c_float(beta), int(bool(reset)), N.stream())
    N.check(rc, "loco_quantize")
    return q, params


def dequantize(q, params, groups, num_bits=8, q_type=Symmetric, dtype=torch.float16):
    sym = q_type == Symmetric
    if q.dim() > 1:
        out = dequantize(q.contiguous().view(-1), params, groups, num_bits, q_type, dtype)
        return out.view(*q.shape[:-1], q.shape[-1] if num_bits == 8 else q.shape[-1] * 2)
    n = q.numel() * (1 if num_bits == 8 else 2)
    gs = n // groups
    if not q.is_cuda:
        return _host_dequant(q, params, groups, num_bits, sym, dtype).reshape(-1)
    out = torch.empty(n, dtype=dtype, device=q.device)
    rc = N.cuda().dsb_dequantize(_p(q), _p(params.contiguous()), _p(out), ctypes.c_int64(groups), gs, num_bits, int(sym),
                                 N.dt(out), N.stream())
    N.check(rc, "dequantize")
    return out


def swizzle_perm(groups, nodes, devices_per_node, device):
    """Output slot of every input group so that partition (node n, device d) lands at (d, n): after the
    intra-node all-to-all each device holds one contiguous piece per node (reference swizzled_quantize.cu)."""
    parts = nodes * devices_per_node
    assert groups % parts == 0
    gpp = groups // parts
    g = torch.arange(groups, device=device, dtype=torch.int64)
    part, within = g // gpp, g % gpp
    n, d = part // devices_per_node, part % devices_per_node
    return ((d * nodes + n) * gpp + within).to(torch.int32)


def swizzle_quant(x, groups, num_bits=8, q_type=Symmetric, pipeline_size=1, nodes=1, devices_per_node=1):
    perm = swizzle_perm(groups, nodes, devices_per_node, x.device) if nodes * devices_per_node > 1 else None
    return quantize(x, groups, num_bits, q_type, group_perm=perm)


def quantized_reduction(q, params, in_groups, out_groups, num_bits=8, q_type=Symmetric, devices_per_node=1,
                        err=None, err_beta=0.0):
    """Dequantize the ``peers = in_groups // out_groups`` chunks in ``q``, sum them and requantize."""
    sym = q_type == Symmetric
    peers = in_groups // out_groups
    n_in = q.numel() * (1 if num_bits == 8 else 2)
    gs = n_in // in_groups
    if not q.is_cuda:
        deq = _host_dequant(q, params, in_groups, num_bits, sym, torch.float32).reshape(peers, out_groups, gs)
        full = torch.zeros(out_groups, gs)
        for p in range(peers):  # the kernel's order of summation
            full = full + deq[p]
        if err is not None:
            e = err.view(out_groups, gs)
            full = _fma32(torch.tensor(err_beta, dtype=torch.float32), e, full)
        oq, op = _host_quant(full, out_groups, num_bits, sym)
        if err is not None:
            ok = torch.isfinite(op.reshape(out_groups, -1)[:, :1])  # a non-finite group leaves its error slice as it was
            e.copy_(torch.where(ok, full - _host_dequant(oq, op, out_groups, num_bits, sym, torch.float32), e))
        return oq.reshape(-1), op
    oq = torch.empty(out_groups * gs // (1 if num_bits == 8 else 2), dtype=torch.int8, device=q.device)
    op = torch.empty(out_groups if sym else out_groups * 2, dtype=torch.float32, device=q.device)
    rc = N.cuda().dsb_dequant_reduce(_p(q), _p(params.contiguous()), _p(oq), _p(op), peers, out_groups, gs, num_bits,
                                     int(sym), _p(err), N.c_f(err_beta), N.stream())
    N.check(rc, "dequant_reduce")
    return oq, (op if sym else op.view(out_groups, 2))


def loco_quantized_reduction(q, params, err, in_groups, out_groups, num_bits=8, q_type=Symmetric, devices_per_node=1,
                             err_beta=0.8):
    return quantized_reduction(q, params, in_groups, out_groups, num_bits, q_type, devices_per_node, err=err,
                               err_beta=err_beta)


def fake_quantize(x, groups, num_bits, q_type=Symmetric, stochastic=False, seed=0):
    """In-place quantize-dequantize (MoQ / QAT).  Reference: ``ds_quantize_*`` / ``ds_sr_quantize_*``."""
    sym = q_type == Symmetric
    gs = x.numel() // groups
    if not x.is_cuda:
        v, sc, lo = _host_codes(x.reshape(groups, gs).float(), num_bits, sym, stochastic)
        x.copy_(_fma32(v, sc, lo).reshape(x.shape).to(x.dtype))
        return x
    rc = N.cuda().dsb_fake_quantize(_p(x), ctypes.c_int64(groups), gs, num_bits, int(sym), N.dt(x), int(stochastic),
                                    ctypes.c_uint32(seed & 0xffffffff), N.stream())
    N.check(rc, "fake_quantize")
    return x


def ds_quantizer(input, groups=1, bit_num=8, sr=False, asym=False):
    """Reference-compatible entry point (``ops/quantizer/quantizer.py:18``)."""
    return fake_quantize(input, groups, bit_num, Asymmetric if asym else Symmetric, stochastic=sr,
                         seed=int(torch.randint(0, 2**31 - 1, (1, )).item()) if sr else 0)


def _binding(sr, asym):

    def fn(vals, groups, bits):
        return ds_quantizer(vals, groups, bits, sr=sr, asym=asym)

    return fn


# the reference extension's entry points (``csrc/quantization/pt_binding.cpp``): one per dtype / rounding / symmetry,
# all in-place quantize-dequantize; here the dtype is read from the tensor
ds_quantize_fp32 = ds_quantize_fp16 = ds_quantize_bf16 = _binding(False, False)
ds_sr_quantize_fp32 = ds_sr_quantize_fp16 = ds_sr_quantize_bf16 = _binding(True, False)
ds_quantize_asym_fp32 = ds_quantize_asym_fp16 = ds_quantize_asym_bf16 = _binding(False, True)
ds_sr_quantize_asym_fp32 = ds_sr_quantize_asym_fp16 = ds_sr_quantize_asym_bf16 = _binding(True, True)


class Quantizer:
    """Object API used by ZeRO++ (reference ``CUDAQuantizer``, partition_parameters.py:769)."""

    def __init__(self, q_bits=8, q_type=Symmetric, group_size=2048):
        self.q_bits, self.q_type, self.group_size = q_bits, q_type, group_size

    def groups_for(self, numel):
        g = max(1, numel // self.group_size)
        while numel % g:
            g -= 1
        return g

    def quantize(self, x, groups=None):
        groups = groups or self.groups_for(x.numel())
        return quantize(x, groups, self.q_bits, self.q_type)

    def dequantize(self, q, params, dtype=torch.bfloat16):
        groups = params.shape[0]
        return dequantize(q, params, groups, self.q_bits, self.q_type, dtype)


def loco_swizzle_quant(x, err, groups, num_bits=8, q_type=Symmetric, pipeline_size=1, nodes=1, devices_per_node=1, err_beta=0.8):
    """LoCo variant of :func:`swizzle_quant`: quantise ``x + err`` and fold the new quantisation error back into ``err``
    (exponential average) so it is re-injected next step (reference ``loco_swizzle_quant``)."""
    comp = x.float() + err
    q, params = swizzle_quant(comp.to(x.dtype), groups, num_bits, q_type, pipeline_size, nodes, devices_per_node)
    deq = fake_quantize(comp.to(x.dtype).contiguous().view(-1), groups, num_bits, q_type).view_as(comp).float()
    err.mul_(err_beta).add_(comp - deq, alpha=1 - err_beta)
    return q, params
