"""Symmetric-memory context: segments mapped on every rank + the in-kernel NVLink collectives.

Python face of ``csrc/cuda/symm_mem.cpp`` (VMM allocation, fd exchange, peer mapping, NVLS multicast)
and ``csrc/cuda/symm_coll.cu`` (all-gather, reduce-scatter fused with scale+accumulate / Adam, one-shot
all-reduce, device barrier).  See ``comm/symm.py`` for the role of this layer.

Allocation is *collective*: every rank of the group must call :meth:`SymmContext.alloc` with the same
sizes in the same order (ZeRO initialisation does), so an allocation lives at the same offset of the same
segment on every rank and a peer address is simply ``peer_base[p] + (ptr - local_base)``.
"""
import ctypes
import os
import uuid
from typing import List, Optional

import torch
import torch.distributed as dist

from deepspeed_b200.ops import native as N
from deepspeed_b200.utils.logging import logger

CH_BARRIER, CH_AG, CH_RS, CH_AR = 0, 1, 2, 3
_DEFAULT_SEGMENT = int(os.environ.get("DSB200_SYMM_SEGMENT_MB", "1024")) << 20


def _lib():
    lib = N.cuda()
    lib.dsb_symm_granularity.restype = ctypes.c_int64
    return lib


def probe(group=None):
    """Can ``group`` use symmetric memory?  Single node, <= 8 ranks, VMM + fd handles supported."""
    if not torch.cuda.is_available():
        return False, "no CUDA device"
    if not dist.is_initialized():
        return False, "torch.distributed not initialised"
    world = dist.get_world_size(group)
    if world < 2:
        return False, "world size 1"
    lib = _lib()
    if world > lib.dsb_symm_max_ranks():
        return False, f"world {world} > {lib.dsb_symm_max_ranks()}"
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("LOCAL_SIZE", dist.get_world_size())))
    if local_world < dist.get_world_size():
        return False, "multi-node job (peer mapping is intra-node)"
    caps = lib.dsb_symm_caps(torch.cuda.current_device())
    if not (caps & 1):
        return False, "driver lacks VMM / POSIX-fd handle support"
    ok = torch.tensor([1], device="cuda", dtype=torch.int32)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
    return bool(ok.item()), "a peer cannot map memory"


class _Raw:
    """Expose a raw device range through the CUDA array interface so torch can alias it."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes, ), "typestr": "|u1", "data": (ptr, False), "version": 3}


class _Segment:

    def __init__(self, ctx: "SymmContext", nbytes: int, want_mc: bool):
        lib = ctx.lib
        dev = ctx.device_index
        self.nbytes = nbytes
        ptr, handle, fd = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int(-1)
        rc = lib.dsb_symm_alloc(dev, ctypes.c_int64(nbytes), ctypes.byref(ptr), ctypes.byref(handle), ctypes.byref(fd))
        if rc != 0:
            raise RuntimeError(f"dsb_symm_alloc failed: {rc}")
        self.local_ptr, self.handle = ptr.value, handle.value
        fds = (ctypes.c_int * ctx.world)()
        tag = ctx.next_tag()
        rc = lib.dsb_exchange_fds(tag.encode(), ctx.rank, ctx.world, fd.value, fds, 120)
        lib.dsb_close_fd(fd.value)
        if rc != 0:
            raise RuntimeError(f"fd exchange failed: {rc}")
        self.peer_ptrs: List[int] = []
        self.peer_handles: List[int] = []
        for r in range(ctx.world):
            if r == ctx.rank:
                self.peer_ptrs.append(self.local_ptr)
                self.peer_handles.append(0)
            else:
                p, h = ctypes.c_uint64(), ctypes.c_uint64()
                rc = lib.dsb_symm_import(dev, fds[r], ctypes.c_int64(nbytes), ctypes.byref(p), ctypes.byref(h))
                if rc != 0:
                    raise RuntimeError(f"dsb_symm_import(rank {r}) failed: {rc}")
                self.peer_ptrs.append(p.value)
                self.peer_handles.append(h.value)
            lib.dsb_close_fd(fds[r])
        self.mc_ptr = 0
        if want_mc:
            self._try_multicast(ctx)
        self.tensor = torch.as_tensor(_Raw(self.local_ptr, nbytes), device=f"cuda:{dev}")
        self.offset = 0

    def _try_multicast(self, ctx):
        lib, dev = ctx.lib, ctx.device_index
        ok = 1
        mc_handle = ctypes.c_uint64(0)
        fd = ctypes.c_int(-1)
        try:
            if ctx.rank == 0:
                if lib.dsb_mc_create(ctx.world, ctypes.c_int64(self.nbytes), ctypes.byref(mc_handle),
                                     ctypes.byref(fd)) != 0:
                    ok = 0
            # every rank takes part in the exchange (non-zero ranks send a placeholder descriptor)
            send_fd = fd.value if (ctx.rank == 0 and ok) else os.open("/dev/null", os.O_RDONLY)
            fds = (ctypes.c_int * ctx.world)()
            rc = lib.dsb_exchange_fds(ctx.next_tag().encode(), ctx.rank, ctx.world, send_fd, fds, 120)
            if ctx.rank != 0:
                os.close(send_fd)
            if rc != 0:
                ok = 0
            if ok and ctx.rank != 0:
                if lib.dsb_mc_import(fds[0], ctypes.byref(mc_handle)) != 0:
                    ok = 0
            for r in range(ctx.world):
                lib.dsb_close_fd(fds[r])
            if ctx.rank == 0 and fd.value >= 0:
                lib.dsb_close_fd(fd.value)
            if ok and lib.dsb_mc_add_device(mc_handle, dev) != 0:
                ok = 0
        except Exception as e:  # pragma: no cover
            logger.warning(f"multicast setup raised {e!r}")
            ok = 0
        t = torch.tensor([ok], device="cuda", dtype=torch.int32)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=ctx.group)  # also orders add_device before bind
        if not int(t.item()):
            return
        mc_ptr = ctypes.c_uint64(0)
        rc = lib.dsb_mc_bind_and_map(mc_handle, ctypes.c_uint64(self.handle), dev, ctypes.c_int64(self.nbytes),
                                     ctypes.byref(mc_ptr))
        t = torch.tensor([1 if rc == 0 else 0], device="cuda", dtype=torch.int32)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=ctx.group)
        if int(t.item()):
            self.mc_ptr = mc_ptr.value

    def contains(self, ptr: int) -> bool:
        return self.local_ptr <= ptr < self.local_ptr + self.nbytes


class SymmContext:

    def __init__(self, group=None):
        self.group = group
        self.lib = _lib()
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device_index = torch.cuda.current_device()
        self.caps = self.lib.dsb_symm_caps(self.device_index)
        nvls_env = os.environ.get("DSB200_NVLS", "auto")
        self.want_mc = bool(self.caps & 2) and nvls_env != "0"
        self.gran = int(self.lib.dsb_symm_granularity(self.device_index, self.world, int(self.want_mc)))
        if self.gran <= 0:
            raise RuntimeError("cannot query allocation granularity")
        # one job-unique prefix for the abstract unix socket names
        obj = [uuid.uuid4().hex[:12] if self.rank == 0 else None]
        dist.broadcast_object_list(obj, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        self._prefix = f"dsb200-{obj[0]}"
        self._tag = 0
        self.segments: List[_Segment] = []
        self.epochs = [1] * self.lib.dsb_symm_channels()
        # CTAs given to the fused reduce-scatter(+Adam) kernels: each rank reduces and steps 1/world of every unit, so small
        # worlds need more CTAs per kernel to keep up with backward (measured on Llama-3-8B: 2 GPUs 394.8 ms @64 -> 390.1 ms
        # @128; 8 GPUs prefer 64, which leaves more SM issue slots to the concurrent GEMMs)
        self.ctas = int(os.environ.get("DSB200_SYMM_CTAS", "128" if self.world <= 2 else "64"))
        # the LAST reduction of a backward pass has no GEMM left to share the SMs with: give it the whole chip
        self.tail_ctas = int(os.environ.get("DSB200_SYMM_TAIL_CTAS", "148"))
        self.ag_ctas = int(os.environ.get("DSB200_SYMM_AG_CTAS", str(self.ctas)))
        self.ag_mode = os.environ.get("DSB200_SYMM_AG", "ce").lower()  # "ce" (DMA engines) | "kernel" (SM pull)
        # signal pads live in their own small segment (never multicast-bound)
        self._pad_seg = _Segment(self, self._round(max(self.lib.dsb_symm_pad_bytes(), 4096)), want_mc=False)
        self._pad_seg.tensor.zero_()
        torch.cuda.synchronize()
        dist.barrier(group=group)
        self._pads = (ctypes.c_void_p * self.world)(*[ctypes.c_void_p(p) for p in self._pad_seg.peer_ptrs])
        self._partials = None
        logger.info(f"symmetric memory up: world={self.world} granularity={self.gran >> 20} MiB "
                    f"nvls={'yes' if self.want_mc else 'no'}")

    # ---- allocation -----------------------------------------------------------------------------
    def next_tag(self):
        self._tag += 1
        return f"{self._prefix}-{self._tag}"

    def _round(self, n):
        return (n + self.gran - 1) // self.gran * self.gran

    def alloc(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        """Collective: all ranks must allocate the same sequence of sizes."""
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        nbytes_al = (nbytes + 255) // 256 * 256
        seg = self.segments[-1] if self.segments else None
        if seg is None or seg.offset + nbytes_al > seg.nbytes:
            seg = _Segment(self, self._round(max(nbytes_al, _DEFAULT_SEGMENT)), self.want_mc)
            self.segments.append(seg)
        t = seg.tensor[seg.offset:seg.offset + nbytes].view(dtype)
        seg.offset += nbytes_al
        return t

    def _seg_of(self, ptr: int) -> Optional[_Segment]:
        for s in self.segments:
            if s.contains(ptr):
                return s
        return None

    def owns(self, t: torch.Tensor) -> bool:
        return t is not None and t.is_cuda and self._seg_of(t.data_ptr()) is not None

    def _peers(self, t: torch.Tensor, elem_offset: int = 0):
        seg = self._seg_of(t.data_ptr())
        off = t.data_ptr() - seg.local_ptr + elem_offset * t.element_size()
        arr = (ctypes.c_void_p * self.world)(*[ctypes.c_void_p(p + off) for p in seg.peer_ptrs])
        mc = ctypes.c_void_p(seg.mc_ptr + off) if seg.mc_ptr else ctypes.c_void_p(0)
        return arr, mc

    def _take_epochs(self, ch, n):
        e = self.epochs[ch]
        self.epochs[ch] = (e + n) & 0x7fffffff or 1
        return ctypes.c_uint32(e)

    # ---- collectives ---------------------------------------------------------------------------------
    def barrier(self):
        """Device-side barrier on the current stream (no host sync)."""
        rc = self.lib.dsb_symm_barrier(self._pads, self.rank, self.world, CH_BARRIER, self._take_epochs(CH_BARRIER, 1),
                                       N.stream())
        N.check(rc, "symm_barrier")

    def all_gather(self, full: torch.Tensor, shard: torch.Tensor, shard_numel: int):
        """``full[p*S:(p+1)*S] = shard_of_rank_p``; ``shard`` must live at the same symmetric offset on
        every rank.  No internal barrier: callers order it after the optimizer-step barrier."""
        shards, _ = self._peers(shard)
        nbytes = shard_numel * shard.element_size()
        if self.ag_mode == "ce":
            # copy-engine DMA straight from the peers' shards: no SMs taken from the GEMMs it overlaps with
            rc = self.lib.dsb_symm_all_gather_ce(shards, N.ptr(full), ctypes.c_int64(nbytes), self.rank, self.world,
                                                 N.stream())
            N.check(rc, "symm_all_gather_ce")
            return
        rc = self.lib.dsb_symm_all_gather(shards, N.ptr(full), ctypes.c_int64(nbytes), self._pads, self.rank, self.world,
                                          CH_AG, ctypes.c_uint32(0), 0, self.ag_ctas, N.stream())
        N.check(rc, "symm_all_gather")

    def all_gather_matmul(self, a, full, shard, shard_numel, w_offset, n_rows, k, chunk_bytes=1 << 20, comm_ctas=32):
        """``a [M,K] @ W^T`` where ``W [n_rows, K]`` lives ``w_offset`` elements into the gathered unit buffer
        ``full`` — ONE kernel that pulls every rank's shard over NVLink (trailing ``comm_ctas`` CTAs, chunk flags
        with release/acquire) while the wgmma tiles of rows that already arrived are being multiplied.
        Returns ``(out [M, n_rows])``; on return-to-stream the whole unit is resident in ``full``."""
        from deepspeed_b200.ops.kernels import gemm_sm100
        shards, _ = self._peers(shard)
        nbytes = shard_numel * shard.element_size()
        while nbytes % chunk_bytes:
            chunk_bytes //= 2
        n_chunks = (nbytes // chunk_bytes) * self.world
        if getattr(self, "_agmm_flags", None) is None or self._agmm_flags.numel() < n_chunks:
            self._agmm_flags = torch.zeros(max(n_chunks, 4096), dtype=torch.int32, device="cuda")
            self._agmm_epoch = 0
        self._agmm_epoch = (self._agmm_epoch + 1) & 0x7fffffff or 1
        w_view = full[w_offset:w_offset + n_rows * k].view(n_rows, k)
        return gemm_sm100.matmul_nt_allgather(a, w_view, full, [int(x or 0) for x in shards], self._agmm_flags, nbytes,
                                              chunk_bytes, w_offset * full.element_size(), self.world, self.rank,
                                              self._agmm_epoch, comm_ctas=comm_ctas)

    def _sumsq_buf(self):
        if self._partials is None:
            self._partials = torch.zeros(max(self.ctas, 256), dtype=torch.float32, device="cuda")
        return self._partials

    def reduce_scatter_accumulate(self, full_g: torch.Tensor, dst: torch.Tensor, shard_numel: int, scale: float,
                                  accumulate: bool, tail: bool = False):
        grads, mc = self._peers(full_g)
        if os.environ.get("DSB200_NVLS_RS", "1") == "0":
            mc = ctypes.c_void_p(0)
        rc = self.lib.dsb_symm_reduce_scatter_acc(grads, mc, N.ptr(dst), ctypes.c_int64(shard_numel), N.dt(full_g),
                                                  N.dt(dst), N.c_f(scale), int(accumulate), self._pads, self.rank,
                                                  self.world, CH_RS, self._take_epochs(CH_RS, 2), ctypes.c_void_p(0),
                                                  max(self.ctas, self.tail_ctas) if tail else self.ctas, N.stream())
        N.check(rc, "symm_reduce_scatter_acc")

    def reduce_scatter_adam(self, zo, rt, full_g: torch.Tensor, scale: float, tail: bool = False):
        """Reduce-scatter fused with the AdamW update of this rank's shard of unit ``rt``."""
        u = rt.u
        a = u.arena_offset
        segs = []
        for (prt, gi, s0, e0) in zo.pieces:
            if prt is not rt or gi < 0:
                continue
            g = zo.param_groups[gi]
            b1, b2 = g.get("betas", zo.flat_opt.defaults["betas"])
            step = zo.group_steps[gi] + 1
            bc = g.get("bias_correction", True)
            segs.append(_AdamSeg(s0 - a, e0 - a, g["lr"], b1, b2, g.get("eps", zo.flat_opt.defaults["eps"]),
                                 g.get("weight_decay", 0.0), 1.0 - b1**step if bc else 1.0,
                                 1.0 - b2**step if bc else 1.0, int(zo.flat_opt.adamw)))
        arr = (_AdamSeg * max(len(segs), 1))(*segs)
        grads, mc = self._peers(full_g)
        if os.environ.get("DSB200_NVLS_RS", "1") == "0":
            mc = ctypes.c_void_p(0)
        st = zo.flat_opt.state_tensors()
        n = u.shard_numel
        lp = zo._lp_shard(u)
        rc = self.lib.dsb_symm_reduce_scatter_adam(grads, mc, N.ptr(zo.master[a:a + n]), N.ptr(st["exp_avg"][a:a + n]),
                                                   N.ptr(st["exp_avg_sq"][a:a + n]), N.ptr(lp), ctypes.c_int64(n),
                                                   N.dt(full_g), N.dt(lp), N.c_f(scale), arr, len(segs), self._pads,
                                                   self.rank, self.world, CH_RS, self._take_epochs(CH_RS, 2),
                                                   max(self.ctas, self.tail_ctas) if tail else self.ctas, N.stream())
        N.check(rc, "symm_reduce_scatter_adam")

    def all_reduce_(self, t: torch.Tensor) -> bool:
        """One-shot sum all-reduce of a symmetric tensor (numel multiple of 8), in place."""
        if t.numel() % 8 or not t.is_contiguous():
            return False
        bufs, _ = self._peers(t)
        out = torch.empty_like(t)
        rc = self.lib.dsb_symm_all_reduce(bufs, N.ptr(out), ctypes.c_int64(t.numel()), N.dt(t), self._pads, self.rank,
                                          self.world, CH_AR, self._take_epochs(CH_AR, 2), min(self.ctas, 16), N.stream())
        N.check(rc, "symm_all_reduce")
        t.copy_(out)
        return True

    def close(self):
        torch.cuda.synchronize()
        for seg in self.segments + [self._pad_seg]:
            for r, (p, h) in enumerate(zip(seg.peer_ptrs, seg.peer_handles)):
                if r != self.rank and p:
                    self.lib.dsb_symm_unmap(ctypes.c_uint64(p), ctypes.c_uint64(h), ctypes.c_int64(seg.nbytes))
        self.segments.clear()


class _AdamSeg(ctypes.Structure):
    _fields_ = [("start", ctypes.c_int64), ("end", ctypes.c_int64), ("lr", ctypes.c_float), ("beta1", ctypes.c_float),
                ("beta2", ctypes.c_float), ("eps", ctypes.c_float), ("wd", ctypes.c_float), ("bc1", ctypes.c_float),
                ("bc2", ctypes.c_float), ("adamw", ctypes.c_int)]
