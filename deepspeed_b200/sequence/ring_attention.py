"""Ring / context-parallel attention (absent from the reference, SURVEY.md 5.7 -- added natively).

Each rank owns a contiguous sequence block of Q, K, V.  K/V blocks travel around the ring (P-1 hops of
``batch_isend_irecv``); after every hop the local Q attends to the visiting block and the partial results are
merged with the log-sum-exp rule (same online-softmax algebra as ``fpdt_layer.update_out_and_lse``).  Causal
masking skips blocks from the future and applies the triangular mask only on the diagonal block.  On an
NVSwitch box every hop is a full-bandwidth peer copy, so the ring is bandwidth-equivalent to an all-gather of
K/V but keeps the memory footprint at two blocks.
"""
import math

import torch

from deepspeed_b200 import comm as dist


class _RingAttention(torch.autograd.Function):
    """Per-hop attention and its backward run on the framework's pair kernels (``fpdt_layer._pair_fwd / _pair_bwd``: wgmma
    flash attention for head dim 128 / bf16, the register-accumulator kernels for head dims 16-64, fp32 PyTorch otherwise);
    like FPDT, the backward of every (local Q, visiting K/V) pair uses the FINAL output and log-sum-exp of the local queries,
    so the pair contributions simply add and nothing is recomputed in forward mode."""

    @staticmethod
    def forward(ctx, q, k, v, group, causal, scale):
        from deepspeed_b200.sequence.fpdt_layer import _merge, _pair_fwd
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        scale = scale or 1.0 / math.sqrt(q.shape[-1])
        qs, kb, vb = (t.permute(0, 2, 1, 3).contiguous() for t in (q, k, v))  # [B, S, H, D] blocks travel the ring
        out = lse = None
        src = rank
        for hop in range(world):
            if not causal or src <= rank:
                o2, l2 = _pair_fwd(qs, kb, vb, causal and src == rank, scale)
                out, lse = _merge(out, lse, o2, l2)
            if hop < world - 1:
                kb, vb = _rotate(kb, vb, group, rank, world)
                src = (src - 1) % world
        o = out.to(q.dtype)
        ctx.save_for_backward(qs, k, v, o, lse)
        ctx.group, ctx.causal, ctx.scale = group, causal, scale
        return o.permute(0, 2, 1, 3)

    @staticmethod
    def backward(ctx, dout):
        from deepspeed_b200.sequence.fpdt_layer import _pair_bwd
        qs, k, v, o, lse = ctx.saved_tensors
        group, causal, scale = ctx.group, ctx.causal, ctx.scale
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        do = dout.permute(0, 2, 1, 3).contiguous()
        kb, vb = (t.permute(0, 2, 1, 3).contiguous() for t in (k, v))
        dq = torch.zeros(qs.shape, dtype=torch.float32, device=qs.device)
        dkb = torch.zeros(kb.shape, dtype=torch.float32, device=kb.device)
        dvb = torch.zeros(vb.shape, dtype=torch.float32, device=vb.device)
        src = rank
        for hop in range(world):
            if not causal or src <= rank:
                dq_i, dk_i, dv_i = _pair_bwd(do, qs, kb, vb, o, lse, causal and src == rank, scale)
                dq += dq_i
                dkb += dk_i
                dvb += dv_i
            # the K/V block travels on together with its gradient accumulators; after P hops both are home
            if world > 1:
                kb, vb, dkb, dvb = _rotate4(kb, vb, dkb, dvb, group, rank, world)
            src = (src - 1) % world
        back = lambda t, like: t.to(like.dtype).permute(0, 2, 1, 3)
        return back(dq, qs), back(dkb, k), back(dvb, v), None, None, None


def _rotate(a, b, group, rank, world):
    nxt = dist.get_global_rank(group, (rank + 1) % world)
    prv = dist.get_global_rank(group, (rank - 1) % world)
    ra, rb = torch.empty_like(a), torch.empty_like(b)
    ops = [dist.P2POp(torch.distributed.isend, a, nxt, group), dist.P2POp(torch.distributed.isend, b, nxt, group),
           dist.P2POp(torch.distributed.irecv, ra, prv, group), dist.P2POp(torch.distributed.irecv, rb, prv, group)]
    for w in dist.batch_isend_irecv(ops):
        w.wait()
    return ra, rb


def _rotate4(a, b, c, d, group, rank, world):
    a2, b2 = _rotate(a, b, group, rank, world)
    c2, d2 = _rotate(c.contiguous(), d.contiguous(), group, rank, world)
    return a2, b2, c2, d2


def ring_attention(q, k, v, group=None, causal=True, scale=None):
    """q, k, v: ``[B, H, S_local, D]`` (this rank's contiguous sequence block)."""
    if dist.get_world_size(group) == 1:
        return torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=scale)
    return _RingAttention.apply(q, k, v, group, causal, scale)
