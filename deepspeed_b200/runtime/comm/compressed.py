"""Error-compensated 1-bit all-reduce (the collective under 1-bit Adam / 0-1 Adam / 1-bit LAMB).

Role parity: reference ``runtime/comm/{nccl,mpi,hccl,compressed}.py`` ``compressed_allreduce``.  Two-phase
scheme: every worker sends the *sign bits* (+ one fp32 scale) of its error-compensated buffer; rank r acts as
the server of chunk r, averages what it received, compresses the average again (with its own error feedback)
and all-gathers the result.  Bits are packed 8-per-byte with torch integer ops (the reference uses cupy
``packbits``), so the wire volume is 1/32 of fp32.
"""
import torch

from deepspeed_b200 import comm as dist

_POW2 = None


def _pow2(device):
    global _POW2
    if _POW2 is None or _POW2.device != device:
        _POW2 = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.uint8, device=device)
    return _POW2


def pack_signs(x: torch.Tensor) -> torch.Tensor:
    """bool/sign of ``x`` (>=0 -> 1) packed MSB-first into uint8; ``x.numel()`` must be a multiple of 8."""
    bits = (x >= 0).view(-1, 8).to(torch.uint8)
    return (bits * _pow2(x.device)).sum(dim=1, dtype=torch.uint8)


def unpack_signs(packed: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """uint8 -> +-1 values of length ``8 * packed.numel()``."""
    bits = (packed.view(-1, 1) & _pow2(packed.device)).ne(0)
    return bits.to(dtype).mul_(2).sub_(1).view(-1)


def _native(t):
    return t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()


def compress_with_feedback(work: torch.Tensor, error_out: torch.Tensor):
    """``work`` (already holding value + previous error) -> ``(packed signs, scale)``; writes the new error
    ``work - scale * sign(work)`` into ``error_out``.  One fused sm_90a pass on the device (``misc.cu onebit_pack``)."""
    scale = work.norm() / (work.numel()**0.5)
    if _native(work) and _native(error_out) and work.numel() % 8 == 0:
        from deepspeed_b200.ops import native as N
        packed = torch.empty(work.numel() // 8, dtype=torch.uint8, device=work.device)
        rc = N.cuda().dsb_onebit_pack(N.ptr(work), N.ptr(scale.reshape(1)), N.ptr(packed), N.ptr(error_out),
                                      N.c_i64(work.numel()), N.stream())
        N.check(rc, "onebit_pack")
        return packed, scale
    packed = pack_signs(work)
    error_out.copy_(work - scale * unpack_signs(packed, work.dtype))
    return packed, scale


def decompress_average(packed: torch.Tensor, scales: torch.Tensor, n: int) -> torch.Tensor:
    """``packed [R, n/8]`` sign bytes + ``scales [R]`` -> mean over the R senders of ``scale_r * sign_r`` (length n)."""
    R = scales.numel()
    if packed.is_cuda and packed.is_contiguous() and scales.dtype == torch.float32 and n % 8 == 0:
        from deepspeed_b200.ops import native as N
        out = torch.empty(n, dtype=torch.float32, device=packed.device)
        rc = N.cuda().dsb_onebit_unpack_avg(N.ptr(packed), N.ptr(scales.contiguous()), N.ptr(out), N.c_i64(n), R,
                                            N.c_f(1.0 / R), N.stream())
        N.check(rc, "onebit_unpack_avg")
        return out
    vals = unpack_signs(packed.reshape(-1), torch.float32).view(R, n)
    return (vals * scales.view(R, 1).float()).sum(0).div_(R)


class CompressedBackend:

    def __init__(self, mpu=None, group=None):
        if mpu is not None:
            self.world_group = mpu.get_data_parallel_group()
        else:
            self.world_group = group
        self.rank = dist.get_rank(self.world_group)
        self.size = dist.get_world_size(self.world_group)

    def my_igather(self, rank, size, group, sendbuf, recvbuf, root):
        if rank == root:
            recvbuf[rank].copy_(sendbuf)
            reqs = [dist.irecv(recvbuf[i], src=i, group=group) for i in range(size) if i != rank]
        else:
            reqs = [dist.isend(sendbuf, dst=root, group=group)]
        return reqs

    def compressed_allreduce(self, buffer_m: torch.Tensor, worker_error, server_error, local_rank=None):
        """In: any-shape fp tensor; out: same shape, the (lossy) average over ranks.  ``worker_error`` has the
        padded length (multiple of 8*size), ``server_error`` that length / size."""
        shape = buffer_m.shape
        flat = buffer_m.reshape(-1)
        n = flat.numel()
        padded = worker_error.numel()
        size = self.size
        chunk = padded // size
        assert padded % (8 * size) == 0 and server_error.numel() == chunk
        if padded != n:
            work = torch.zeros(padded, dtype=flat.dtype, device=flat.device)
            work[:n] = flat
        else:
            work = flat.clone()
        # ---- worker compression
        work.add_(worker_error)
        signs, w_scale = compress_with_feedback(work, worker_error)
        # ---- exchange: chunk r of everyone's signs goes to rank r
        send = signs.view(size, chunk // 8)
        recv = torch.empty_like(send)
        if size > 1:
            dist.all_to_all_single(recv.view(-1), send.contiguous().view(-1), group=self.world_group)
            scales = [torch.empty_like(w_scale.view(1)) for _ in range(size)]
            dist.all_gather(scales, w_scale.view(1), group=self.world_group)
            scales = torch.cat(scales)
        else:
            recv.copy_(send)
            scales = w_scale.view(1)
        # ---- server: average, compress again
        server = decompress_average(recv.contiguous(), scales.float(), chunk).to(work.dtype)
        server.add_(server_error)
        s_signs, s_scale = compress_with_feedback(server, server_error)
        # ---- broadcast result
        if size > 1:
            all_signs = [torch.empty_like(s_signs) for _ in range(size)]
            dist.all_gather(all_signs, s_signs, group=self.world_group)
            all_scales = [torch.empty_like(s_scale.view(1)) for _ in range(size)]
            dist.all_gather(all_scales, s_scale.view(1), group=self.world_group)
            out = torch.cat([unpack_signs(sg, work.dtype) * sc for sg, sc in zip(all_signs, all_scales)])
        else:
            out = unpack_signs(s_signs, work.dtype) * s_scale
        return out[:n].view(shape).to(buffer_m.dtype)


NcclBackend = CompressedBackend
MpiBackend = CompressedBackend
HcclBackend = CompressedBackend
