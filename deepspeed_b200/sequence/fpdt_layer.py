"""FPDT / Ulysses-Offload: chunked sequence pipeline with online-softmax merging and a double-buffered host offload.

Parity target: reference ``sequence/fpdt_layer.py`` (``update_out_and_lse :58``, ``FPDT_InputConstruct :79``,
``_FPDTGPUAttentionImpl_ :134``, ``_FPDTGPUOffloadingAttentionImpl_ :510``, ``SequenceChunk :462``,
``FPDT_Attention :971``, ``FPDT_FFN :1056``, ``FPDT_LogitsLoss :1137``).

The local sequence is split into ``num_chunks`` chunks.  Chunk ``i`` is projected, the Ulysses all-to-all trades heads for
sequence, and the chunk attends to key / value chunks ``0..i`` (causal only on the diagonal pair); partial outputs are
merged with the running log-sum-exp.  The whole thing is ONE autograd function (``_FPDTAttentionCore``) with a manual
backward, like the reference: q / k / v / o chunks are parked in a chunk store -- pinned host memory when offloading,
written on a device->host stream and prefetched one pair ahead on a host->device stream -- and the backward walks the
query chunks from last to first, calling the per-pair flash backward with the GLOBAL log-sum-exp of the query chunk, so no
pair is recomputed in forward mode and device memory holds O(chunk) activations for arbitrarily long sequences.

The per-pair kernels are the framework's own: head dim 128 / bf16 -> the wgmma flash attention (``attn_sm90.cu``, returns
LSE, takes it back in backward), head dim 16 / 32 / 64 -> the register-accumulator kernels of ``attn_bias.cu``; anything
else (CPU, fp32) uses the fp32 PyTorch formulation below.
"""
import math
from typing import Optional

import torch
import torch.nn.functional as F

from deepspeed_b200 import comm as dist
from deepspeed_b200.sequence.layer import single_all_to_all, _SeqAllToAll, apply_rotary_pos_emb


def update_out_and_lse(out, lse, block_out, block_lse):
    """Merge two partial attention results over disjoint key sets (all fp32, lse shape [..., S, 1])."""
    if out is None:
        return block_out.float(), block_lse.float()
    new_lse = lse + F.softplus(block_lse - lse)  # log(exp(lse) + exp(block_lse)), stable
    out = torch.exp(lse - new_lse) * out + torch.exp(block_lse - new_lse) * block_out.float()
    return out, new_lse


def _attn_with_lse(q, k, v, causal, scale):
    """q,k,v [B,H,S,D] -> (out fp32, lse fp32 [B,H,S,1]).  GQA by head repetition."""
    if k.shape[1] != q.shape[1]:
        rep = q.shape[1] // k.shape[1]
        k, v = k.repeat_interleave(rep, dim=1), v.repeat_interleave(rep, dim=1)
    s = torch.matmul(q.float(), k.float().transpose(-1, -2)) * scale
    if causal:
        Sq, Sk = s.shape[-2:]
        s = s.masked_fill(~torch.ones(Sq, Sk, dtype=torch.bool, device=s.device).tril_(diagonal=Sk - Sq), float("-inf"))
    lse = torch.logsumexp(s, dim=-1, keepdim=True)
    return torch.matmul(torch.exp(s - lse), v.float()), lse


# ---- per-pair kernels on [B, s, h, d] ("bshd", contiguous) chunks -------------------------------------------------------
def _pair_backend(q, k):
    d = q.shape[-1]
    if q.is_cuda and q.dtype == torch.bfloat16 and d == 128 and q.shape[1] == k.shape[1] and q.shape[1] % 128 == 0:
        return "sm100"
    if q.is_cuda and q.dtype in (torch.bfloat16, torch.float16) and d in (16, 32, 64):
        return "mma"
    return "torch"


def _rep_kv(q, k, v):
    rep = q.shape[2] // k.shape[2]
    if rep == 1:
        return k, v, 1
    return k.repeat_interleave(rep, dim=2), v.repeat_interleave(rep, dim=2), rep


def _pair_fwd(q, k, v, causal, scale):
    """-> (o [B, s, h, d] in q's dtype, lse fp32 [B, h, s])."""
    B, S, hq, d = q.shape
    be = _pair_backend(q, k)
    if be == "sm100":
        from deepspeed_b200.ops.kernels import attention_sm100 as A
        o, lse = A.fwd(q.view(B * S, hq * d), k.view(B * S, -1), v.view(B * S, -1), B, S, hq, k.shape[2], causal=causal,
                       scale=scale)
        return o.view(B, S, hq, d), lse
    if be == "mma":
        from deepspeed_b200.ops.kernels import attn_bias as AB
        kk, vv, _ = _rep_kv(q, k, v)
        o, lse = AB.forward(q.permute(0, 2, 1, 3), kk.permute(0, 2, 1, 3), vv.permute(0, 2, 1, 3), causal=causal, scale=scale)
        return o.permute(0, 2, 1, 3), lse
    o, lse = _attn_with_lse(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3), causal, scale)
    return o.permute(0, 2, 1, 3).to(q.dtype), lse.squeeze(-1)


def _pair_bwd(d_o, q, k, v, o, lse, causal, scale):
    """Gradients of one (query chunk, key chunk) pair given the query chunk's FINAL output and log-sum-exp (the pair's
    probabilities are ``exp(s - lse)``, so the contributions of all pairs simply add)."""
    B, S, hq, d = q.shape
    be = _pair_backend(q, k)
    if be == "sm100":
        from deepspeed_b200.ops.kernels import attention_sm100 as A
        f = lambda t: t.reshape(B * t.shape[1], -1)
        dq, dk, dv = A.bwd(f(d_o), f(q), f(k), f(v), f(o), lse, B, S, hq, k.shape[2], causal=causal, scale=scale)
        return dq.view(q.shape), dk.view(k.shape), dv.view(v.shape)
    if be == "mma":
        from deepspeed_b200.ops.kernels import attn_bias as AB
        kk, vv, rep = _rep_kv(q, k, v)
        t = lambda x: x.permute(0, 2, 1, 3)
        dq, dk, dv, _, _ = AB.backward(t(d_o), t(q), t(kk), t(vv), t(o), lse, causal=causal, scale=scale)
        dq, dk, dv = t(dq), t(dk), t(dv)
        if rep > 1:
            dk = dk.reshape(B, k.shape[1], k.shape[2], rep, d).sum(3)
            dv = dv.reshape(B, k.shape[1], k.shape[2], rep, d).sum(3)
        return dq, dk, dv
    kk, vv, rep = _rep_kv(q, k, v)
    qf, kf, vf, of, gf = (x.permute(0, 2, 1, 3).float() for x in (q, kk, vv, o, d_o))
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if causal:
        Sq, Sk = s.shape[-2:]
        s = s.masked_fill(~torch.ones(Sq, Sk, dtype=torch.bool, device=s.device).tril_(diagonal=Sk - Sq), float("-inf"))
    p = torch.exp(s - lse.unsqueeze(-1))
    dv = torch.matmul(p.transpose(-1, -2), gf)
    ds = p * (torch.matmul(gf, vf.transpose(-1, -2)) - (gf * of).sum(-1, keepdim=True))
    dq = torch.matmul(ds, kf) * scale
    dk = torch.matmul(ds.transpose(-1, -2), qf) * scale
    dq, dk, dv = (x.permute(0, 2, 1, 3) for x in (dq, dk, dv))
    if rep > 1:
        dk = dk.reshape(B, k.shape[1], k.shape[2], rep, -1).sum(3)
        dv = dv.reshape(B, k.shape[1], k.shape[2], rep, -1).sum(3)
    return dq, dk, dv


def _merge(out, lse, bo, bl):
    """Running merge on bshd outputs: ``out`` fp32 [B, s, h, d], ``lse`` fp32 [B, h, s]."""
    if out is None:
        return bo.float(), bl.float().clone()
    new = torch.logaddexp(lse, bl)
    w_old = torch.exp(lse - new).permute(0, 2, 1).unsqueeze(-1)
    w_new = torch.exp(bl - new).permute(0, 2, 1).unsqueeze(-1)
    return out.mul_(w_old).add_(bo.float() * w_new), new


class _ChunkStore:
    """Where q / k / v / o chunks wait between forward and backward.  Without offloading: a dict of device tensors.  With
    offloading: pinned host copies written on a device->host stream as soon as a chunk is produced; ``prefetch`` starts the
    host->device copy on its own stream and ``get`` makes the compute stream wait for exactly that copy, so while pair
    (i, j) computes, the chunks of pair (i, j+1) are in flight (reference ``SequenceChunk`` + the double buffering of
    ``_FPDTGPUOffloadingAttentionImpl_``, ``fpdt_layer.py:462, :510``)."""

    def __init__(self, offload, device):
        self.offload = bool(offload) and device.type == "cuda"
        self.device = device
        self.dev, self.host, self.ready = {}, {}, {}
        self.bytes_offloaded = 0
        if self.offload:
            self.d2h, self.h2d = torch.cuda.Stream(device), torch.cuda.Stream(device)

    def put(self, key, t, keep_on_device=False):
        if not self.offload:
            self.dev[key] = t
            return
        host = torch.empty(t.shape, dtype=t.dtype, device="cpu", pin_memory=True)
        self.d2h.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.d2h):
            host.copy_(t, non_blocking=True)
        t.record_stream(self.d2h)
        self.host[key] = host
        self.bytes_offloaded += t.numel() * t.element_size()
        if keep_on_device:
            self.dev[key] = t

    def prefetch(self, key):
        if not self.offload or key in self.dev or key not in self.host:
            return
        self.h2d.wait_stream(self.d2h)  # the host copy of this chunk must have landed
        with torch.cuda.stream(self.h2d):
            t = self.host[key].to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.h2d)
        self.dev[key], self.ready[key] = t, ev

    def get(self, key):
        self.prefetch(key)
        ev = self.ready.pop(key, None)
        t = self.dev[key]
        if ev is not None:
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ev)
            t.record_stream(cur)
        return t

    def release(self, key):
        """Drop the device copy (the host copy stays) -- no-op without offloading."""
        if self.offload:
            self.dev.pop(key, None)
            self.ready.pop(key, None)

    def drop(self, key):
        self.dev.pop(key, None)
        self.host.pop(key, None)
        self.ready.pop(key, None)


class _FPDTAttentionCore(torch.autograd.Function):
    """QKV projection -> Ulysses all-to-all -> chunked causal attention -> all-to-all back, chunk by chunk, with a manual
    backward (reference ``_FPDTGPUOffloadingAttentionImpl_``, ``fpdt_layer.py:510``).  Returns the context
    ``[S_local, B, hq * d]`` (the output projection stays outside)."""

    @staticmethod
    def forward(ctx, x, w, b, cfg):
        spg, hq, hkv, d, n_chunks, offload, rope = cfg
        sp = dist.get_world_size(spg) if spg is not None else 1
        S, B, _ = x.shape
        cs = S // n_chunks
        scale = 1.0 / math.sqrt(d)
        need_grad = any(ctx.needs_input_grad[:3])
        store = _ChunkStore(offload, x.device)
        a2a = lambda t: single_all_to_all(t.contiguous(), 2, 0, 1, spg) if sp > 1 else t  # heads -> sequence
        outs, lses = [], []
        for i in range(n_chunks):
            qkv = F.linear(x[i * cs:(i + 1) * cs], w, b)
            q, k, v = torch.split(qkv, [hq * d, hkv * d, hkv * d], dim=-1)
            q, k, v = a2a(q.reshape(cs, B, hq, d)), a2a(k.reshape(cs, B, hkv, d)), a2a(v.reshape(cs, B, hkv, d))
            if rope is not None:  # positions of chunk i after the all-to-all are contiguous: [i * cs * sp, (i + 1) * cs * sp)
                cos, sin = (r[i * cs * sp:(i + 1) * cs * sp] for r in rope)
                q, k = apply_rotary_pos_emb(q, cos, sin), apply_rotary_pos_emb(k, cos, sin)
            q, k, v = (t.permute(1, 0, 2, 3).contiguous() for t in (q, k, v))  # [B, s, h, d]
            store.put(("k", i), k, keep_on_device=True)
            store.put(("v", i), v, keep_on_device=True)
            out = lse = None
            for j in range(i + 1):
                if j + 1 <= i:
                    store.prefetch(("k", j + 1))
                    store.prefetch(("v", j + 1))
                kj, vj = store.get(("k", j)), store.get(("v", j))
                bo, bl = _pair_fwd(q, kj, vj, j == i, scale)
                out, lse = _merge(out, lse, bo, bl)
                store.release(("k", j))
                store.release(("v", j))
            o = out.to(x.dtype)
            if need_grad:
                store.put(("q", i), q)
                store.put(("o", i), o)
                lses.append(lse)
            o = o.permute(1, 0, 2, 3)  # [s, B, h_local, d]
            if sp > 1:
                o = single_all_to_all(o.contiguous(), 0, 2, 1, spg)  # sequence -> heads
            outs.append(o.reshape(cs, B, hq * d))
        ctx.save_for_backward(x, w, b)
        ctx.store, ctx.lses, ctx.cfg = store, lses, cfg
        return torch.cat(outs, dim=0)

    @staticmethod
    def backward(ctx, g):
        from deepspeed_b200.sequence.fpdt_layer import apply_rotary_pos_emb_backward
        x, w, b = ctx.saved_tensors
        spg, hq, hkv, d, n_chunks, offload, rope = ctx.cfg
        store, lses = ctx.store, ctx.lses
        sp = dist.get_world_size(spg) if spg is not None else 1
        S, B, _ = x.shape
        cs = S // n_chunks
        scale = 1.0 / math.sqrt(d)
        dx = torch.empty_like(x)
        dw = torch.zeros(w.shape, dtype=torch.float32, device=w.device)
        db = torch.zeros(b.shape, dtype=torch.float32, device=b.device) if b is not None else None
        dk_acc, dv_acc = {}, {}
        for i in reversed(range(n_chunks)):
            gi = g[i * cs:(i + 1) * cs].reshape(cs, B, hq, d)
            if sp > 1:
                gi = single_all_to_all(gi.contiguous(), 2, 0, 1, spg)
            gi = gi.permute(1, 0, 2, 3).contiguous()
            store.prefetch(("k", i))
            store.prefetch(("v", i))
            qi, oi, lse = store.get(("q", i)), store.get(("o", i)), lses[i]
            dq = None
            for j in range(i, -1, -1):
                if j - 1 >= 0:
                    store.prefetch(("k", j - 1))
                    store.prefetch(("v", j - 1))
                kj, vj = store.get(("k", j)), store.get(("v", j))
                dq_ij, dk_ij, dv_ij = _pair_bwd(gi, qi, kj, vj, oi, lse, j == i, scale)
                dq = dq_ij.float() if dq is None else dq.add_(dq_ij)
                if j in dk_acc:
                    dk_acc[j].add_(dk_ij)
                    dv_acc[j].add_(dv_ij)
                else:
                    dk_acc[j], dv_acc[j] = dk_ij.float(), dv_ij.float()
                store.release(("k", j))
                store.release(("v", j))
            for name in ("q", "o", "k", "v"):
                store.drop((name, i))
            # chunk i's q / k / v gradients are final (only query chunks >= i see key chunk i): undo layout, rope, all-to-all
            parts = []
            for t, rot in ((dq, True), (dk_acc.pop(i), True), (dv_acc.pop(i), False)):
                t = t.to(x.dtype).permute(1, 0, 2, 3)  # [s, B, h_local, d]
                if rot and rope is not None:
                    cos, sin = (r[i * cs * sp:(i + 1) * cs * sp] for r in rope)
                    t = apply_rotary_pos_emb_backward(t, cos, sin)
                if sp > 1:
                    t = single_all_to_all(t.contiguous(), 0, 2, 1, spg)
                parts.append(t.reshape(cs, B, -1))
            dqkv = torch.cat(parts, dim=-1)
            dx[i * cs:(i + 1) * cs] = torch.matmul(dqkv, w)
            d2 = dqkv.reshape(-1, dqkv.shape[-1])
            dw.addmm_(d2.t().float(), x[i * cs:(i + 1) * cs].reshape(-1, x.shape[-1]).float())
            if db is not None:
                db.add_(d2.float().sum(0))
        return dx, dw.to(w.dtype), (db.to(b.dtype) if db is not None else None), None


class _FPDTGPUOffloadingAttentionImpl_:
    """The reference's internal entry point (``fpdt_layer.py:510``) under its own name and ``apply`` signature, for code
    that calls it directly: ``x [S_local, B, hidden]`` in the load-balanced chunk order -> context ``[B, S_local, heads,
    head_dim]``. One implementation serves both variants: ``cpu_offloading`` only decides where idle chunks wait."""

    @staticmethod
    def apply(layernorm_output, attention_mask, inference_params, rotary_pos_emb, spg, scatter_idx, gather_idx, hidden_size,
              projection_size, hidden_size_per_attention_head, kv_projection_size, qkv_linear_weight, qkv_linear_bias, dropout,
              num_chunks_attn=8, cpu_offloading=True):
        assert not dropout, "attention dropout is not supported on the chunked path"
        d = int(hidden_size_per_attention_head)
        hq, hkv = int(projection_size) // d, int(kv_projection_size) // d
        S, B, _ = layernorm_output.shape
        rope = tuple(rotary_pos_emb) if isinstance(rotary_pos_emb, (tuple, list)) else None
        offload = bool(cpu_offloading) and layernorm_output.is_cuda
        cfg = (spg, hq, hkv, d, int(num_chunks_attn), offload, rope)
        ctx = _FPDTAttentionCore.apply(layernorm_output, qkv_linear_weight, qkv_linear_bias, cfg)
        return ctx.view(S, B, hq, d).permute(1, 0, 2, 3)


class _FPDTGPUAttentionImpl_(_FPDTGPUOffloadingAttentionImpl_):

    @staticmethod
    def apply(*a):
        a = list(a) + [8, False][max(0, len(a) - 14):]
        a[15] = False
        return _FPDTGPUOffloadingAttentionImpl_.apply(*a)


class SequenceChunk:
    """A K/V (or Q) chunk that may live on the host; ``load_to_gpu`` is asynchronous on a side stream."""

    def __init__(self, chunk: torch.Tensor, device=None, is_in_use=False):
        self.chunk_shape, self.chunk_dtype = chunk.shape, chunk.dtype
        self.device = device or chunk.device
        if torch.cuda.is_available() and chunk.is_cuda:
            host = torch.empty(chunk.shape, dtype=chunk.dtype, device="cpu", pin_memory=True)
            host.copy_(chunk, non_blocking=True)
            self.cpu_chunk = host
        else:
            self.cpu_chunk = chunk.detach().cpu()
        self.gpu_chunk = chunk if is_in_use else None

    def load_to_gpu(self):
        if self.gpu_chunk is None:
            self.gpu_chunk = self.cpu_chunk.to(self.device, non_blocking=True)

    def get_gpu_chunk(self):
        assert self.gpu_chunk is not None and self.gpu_chunk.device == self.device
        return self.gpu_chunk

    def check_gpu_chunk(self):
        return self.gpu_chunk is not None

    def offload(self):
        self.gpu_chunk = None

    def overwrite_to_cpu(self):
        assert self.gpu_chunk is not None
        self.cpu_chunk.copy_(self.gpu_chunk, non_blocking=True)


class FPDT_InputConstruct(torch.nn.Module):
    """Load-balanced chunk assignment (reference :79): the global sequence is cut into ``sp_size * chunks_per_rank``
    pieces and rank ``r`` takes pieces ``r, r + sp_size, ...`` so every rank owns early *and* late (cheap and expensive
    causal) positions. ``generate()`` returns ``(tokens, labels, loss_mask, attention_mask, position_ids)`` for this rank;
    like the reference the loss mask comes back re-ordered for ALL ranks (rank-major), the other tensors sliced.

    ``args.ds_sequence_parallel_fpdt_chunk_size`` (global tokens per attention chunk) sets the number of chunks per rank;
    ``num_chunks`` gives it directly."""

    def __init__(self, tokens, labels, loss_mask, attention_mask, position_ids, args=None, sp_size=1, sp_rank=0,
                 num_chunks=None):
        super().__init__()
        self.tokens, self.labels, self.loss_mask = tokens, labels, loss_mask
        self.attention_mask, self.position_ids = attention_mask, position_ids
        seq = tokens.shape[1]
        assert seq % sp_size == 0
        if num_chunks is None:
            cs = int(getattr(args, "ds_sequence_parallel_fpdt_chunk_size", seq))
            assert seq % cs == 0
            num_chunks = seq // cs
        local = seq // sp_size
        assert local % num_chunks == 0
        self.num_chunk_per_gpu, self.chunk_size = num_chunks, local // num_chunks
        self.sp_size, self.sp_rank = sp_size, sp_rank
        self.global_seq_len, self.local_seq_len, self.batch_size = seq, local, tokens.shape[0]
        self.device = tokens.device

    def _indices(self, rank):
        n, sp, cs = self.num_chunk_per_gpu, self.sp_size, self.chunk_size
        return torch.cat([torch.arange((c * sp + rank) * cs, (c * sp + rank + 1) * cs) for c in range(n)]).to(self.device)

    def generate(self):
        mine = self._indices(self.sp_rank)
        take = lambda t: None if t is None else t.index_select(1, mine)
        lm = self.loss_mask
        if lm is not None:
            lm = lm.index_select(1, torch.cat([self._indices(r) for r in range(self.sp_size)]))
        return take(self.tokens), take(self.labels), lm, self.attention_mask, take(self.position_ids)

    def __iter__(self):  # ``tokens, labels, ... = FPDT_InputConstruct(...)``
        return iter(self.generate())


class FPDT_Attention(torch.nn.Module):
    """Chunked causal self-attention with fused QKV / output projections (reference :971).

    ``forward(hidden_states [S_local, B, H])`` -> ``[S_local, B, H]``.  ``qkv_linear_weight`` is
    ``[3*H_proj, H]`` laid out ``[q | k | v]``; ``num_heads`` may differ from ``num_kv_heads`` (GQA)."""

    def __init__(self, config=None, first_weight=None, first_bias=None, second_weight=None, second_bias=None,
                 sequence_process_group=None, gather_idx: int = 0, scatter_idx: int = 2, return_bias=True,
                 chunk_size=65536, enable_offloading=True, num_heads=None, num_kv_heads=None, head_dim=None):
        super().__init__()
        self.qkv_linear_weight, self.qkv_linear_bias = first_weight, first_bias
        self.qkv_dense_weight, self.qkv_dense_bias = second_weight, second_bias
        self.spg = sequence_process_group
        self.chunk_size = chunk_size
        self.enable_offloading = enable_offloading
        self.return_bias = return_bias
        self.num_heads = num_heads or getattr(config, "num_attention_heads")
        self.num_kv_heads = num_kv_heads or getattr(config, "num_key_value_heads", self.num_heads)
        hidden = getattr(config, "hidden_size", None) or first_weight.shape[1]
        self.head_dim = head_dim or hidden // self.num_heads

    def forward(self, hidden_states, attention_mask=None, rotary_pos_emb=None, cpu_offloading=None):
        """``rotary_pos_emb``: optional ``(cos, sin)`` tables ``[S_global, 1, 1, rot_dim]`` (NeoX layout), applied to q and k
        chunk by chunk after the all-to-all."""
        S, B, _ = hidden_states.shape
        sp = dist.get_world_size(self.spg) if self.spg is not None else 1
        offload = self.enable_offloading if cpu_offloading is None else cpu_offloading
        offload = bool(offload) and hidden_states.is_cuda
        n_chunks = max(1, math.ceil(S * sp / self.chunk_size))
        while S % n_chunks:
            n_chunks += 1
        rope = tuple(rotary_pos_emb) if rotary_pos_emb is not None else None
        cfg = (self.spg, self.num_heads, self.num_kv_heads, self.head_dim, n_chunks, offload, rope)
        ctx = _FPDTAttentionCore.apply(hidden_states, self.qkv_linear_weight, self.qkv_linear_bias, cfg)
        y = F.linear(ctx, self.qkv_dense_weight, None if self.return_bias else self.qkv_dense_bias)
        if self.return_bias:
            return y, self.qkv_dense_bias
        return y


class FPDT_FFN(torch.nn.Module):
    """MLP evaluated chunk by chunk under activation checkpointing so only one chunk's intermediate
    ``[chunk, B, 4H]`` activation is alive (reference :1056)."""

    def __init__(self, first_weight=None, first_bias=None, second_weight=None, second_bias=None, chunk_size=65536,
                 activation=F.gelu, add_bias=True):
        super().__init__()
        self.w1, self.b1, self.w2, self.b2 = first_weight, first_bias, second_weight, second_bias
        self.chunk_size = chunk_size
        self.activation = activation
        self.add_bias = add_bias

    def _chunk(self, x):
        h = self.activation(F.linear(x, self.w1, self.b1))
        return F.linear(h, self.w2, self.b2 if self.add_bias else None)

    def forward(self, x):
        from torch.utils.checkpoint import checkpoint
        S = x.shape[0]
        outs = []
        for s in range(0, S, self.chunk_size):
            xc = x[s:s + self.chunk_size]
            outs.append(checkpoint(self._chunk, xc, use_reentrant=False) if (torch.is_grad_enabled() and
                                                                             x.requires_grad) else self._chunk(xc))
        y = torch.cat(outs, dim=0)
        return y if self.add_bias else (y, self.b2)


class FPDT_LogitsLoss(torch.nn.Module):
    """Vocabulary projection + cross entropy over token chunks: the ``[tokens, vocab]`` logits never
    materialise (reference :1137).  Backed by the framework's fused chunked kernel path."""

    def __init__(self, lm_head_weight, chunk_size=2048, ignore_index=-100):
        super().__init__()
        self.weight = lm_head_weight
        self.chunk_size = chunk_size
        self.ignore_index = ignore_index

    def forward(self, hidden, labels):
        from deepspeed_b200.ops.linear import chunked_linear_xent
        return chunked_linear_xent(hidden.reshape(-1, hidden.shape[-1]), self.weight, labels.reshape(-1),
                                   chunk=self.chunk_size, ignore_index=self.ignore_index)


# ---- element-wise helpers of the reference module (``fpdt_layer.py:32, :1044-1053``) -----------------------------------
def _rotate_half_backward(x):
    x1, x2 = x.chunk(2, dim=-1)
    return torch.cat((x2, -x1), dim=-1)


def apply_rotary_pos_emb_backward(grad_output, freqs_cos, freqs_sin):
    """Adjoint of ``sequence.layer.apply_rotary_pos_emb``."""
    rot = freqs_cos.shape[-1]
    g, g_pass = grad_output[..., :rot], grad_output[..., rot:]
    g = g * freqs_cos + _rotate_half_backward(g * freqs_sin)
    return g if g_pass.shape[-1] == 0 else torch.cat((g, g_pass), dim=-1)


_GELU_K, _GELU_C = 0.7978845608028654, 0.044715


def bias_gelu(x):
    """tanh-approximated GELU."""
    return 0.5 * x * (1.0 + torch.tanh(_GELU_K * x * (1.0 + _GELU_C * x * x)))


def bias_gelu_back(g, x):
    th = torch.tanh(_GELU_K * x * (1.0 + _GELU_C * x * x))
    d = 0.5 * (1.0 + th) + 0.5 * x * (1.0 - th * th) * _GELU_K * (1.0 + 3.0 * _GELU_C * x * x)
    return d * g
