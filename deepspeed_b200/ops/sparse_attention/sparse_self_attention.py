"""Block-sparse self attention (reference ``ops/sparse_attention/sparse_self_attention.py`` +
Triton ``matmul.py``/``softmax.py``).

H100 formulation: on the GPU (bf16 / fp16, head dim 16 / 32 / 64, power-of-two block >= 16) ONE flash-attention kernel
(``csrc/cuda/attn_bias.cu``) replaces the reference's SDD-matmul -> block softmax -> DSD-matmul chain: the layout is read
inside the kernel, score tiles without any active block are skipped (work scales with the number of non-zero blocks),
inactive blocks inside a tile are masked, and the key-padding / attention masks ride the kernel's two additive-bias slots;
the matching backward kernels give dQ / dK / dV.  The gather + SDPA formulation below remains for CPU / fp32 / other shapes:
rows of the block layout are grouped by their number of visible key blocks and each group is one batched dense problem.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .sparsity_config import SparsityConfig


def block_sparse_attention(q, k, v, layout, block, scale=None, key_padding_mask=None, attn_mask=None,
                           key_padding_mask_mode="add", attn_mask_mode="mul"):
    """q,k,v [B, H, S, D]; layout [H, S/block, S/block] 0/1.  Returns [B, H, S, D]."""
    B, H, S, D = q.shape
    nb = S // block
    scale = scale if scale is not None else D**-0.5
    if _native_ok(q, k, v, block):
        from deepspeed_b200.ops.kernels.attn_bias import biased_attention
        b1 = b2 = None
        if key_padding_mask is not None:
            kpm = key_padding_mask.float().view(B, S)
            b1 = (kpm if key_padding_mask_mode == "add" else (1.0 - kpm) * -10000.0).to(q.dtype)
        if attn_mask is not None:
            am = attn_mask.float().view(1, 1, S, S)
            b2 = (am if attn_mask_mode == "add" else (1.0 - am) * -10000.0).to(q.dtype)
        return biased_attention(q, k, v, b1, b2, layout, block, False, scale)
    lay = layout.to(torch.bool)
    out = torch.zeros_like(q)
    qb = q.view(B, H, nb, block, D)
    kb = k.view(B, H, nb, block, D)
    vb = v.view(B, H, nb, block, D)
    bias_full = None
    if key_padding_mask is not None or attn_mask is not None:
        bias_full = torch.zeros(B, 1, S, S, dtype=torch.float32, device=q.device)
        if key_padding_mask is not None:
            kpm = key_padding_mask.float()
            kpm = kpm if key_padding_mask_mode == "add" else (1.0 - kpm) * -10000.0
            bias_full = bias_full + kpm[:, None, None, :]
        if attn_mask is not None:
            am = attn_mask.float()
            am = am if attn_mask_mode == "add" else (1.0 - am) * -10000.0
            bias_full = bias_full + am
    # group (head, q-block) rows by number of visible blocks so each group is one batched SDPA call
    counts = lay.sum(-1)  # [H, nb]
    for nv in counts.unique().tolist():
        if nv == 0:
            continue
        hs, rs = torch.nonzero(counts == nv, as_tuple=True)  # G rows
        G = hs.numel()
        cols = torch.nonzero(lay[hs, rs], as_tuple=True)[1].view(G, nv)  # [G, nv] visible key blocks
        qg = qb[:, hs, rs]  # [B, G, block, D]
        kg = kb[:, hs[:, None], cols].reshape(B, G, nv * block, D)
        vg = vb[:, hs[:, None], cols].reshape(B, G, nv * block, D)
        bias = None
        if bias_full is not None:
            rows_idx = (rs[:, None] * block + torch.arange(block, device=q.device)[None, :])  # [G, block]
            cols_idx = (cols[:, :, None] * block + torch.arange(block, device=q.device)[None, None, :]).reshape(G, -1)
            bias = bias_full[:, 0][:, rows_idx[:, :, None], cols_idx[:, None, :]].to(q.dtype)  # [B, G, block, nv*block]
        og = F.scaled_dot_product_attention(qg, kg, vg, attn_mask=bias, scale=scale)
        out.view(B, H, nb, block, D)[:, hs, rs] = og
    return out


def _native_ok(q, k, v, block):
    from deepspeed_b200.ops.kernels import attn_bias as AB
    return (AB.supported(q, k, v) and q.shape == k.shape == v.shape and block >= 16 and (block & (block - 1)) == 0
            and q.shape[2] % block == 0)


class SparseSelfAttention(nn.Module):

    def __init__(self, sparsity_config=SparsityConfig(num_heads=4), key_padding_mask_mode="add", attn_mask_mode="mul",
                 max_seq_length=2048):
        super().__init__()
        self.sparsity_config = sparsity_config
        self.register_buffer("master_layout", self.sparsity_config.make_layout(max_seq_length))
        self._need_layout_synchronization = True
        self.key_padding_mask_mode = key_padding_mask_mode
        self.attn_mask_mode = attn_mask_mode

    def get_layout(self, L):
        if self._need_layout_synchronization and torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.broadcast(self.master_layout, src=0)
            self._need_layout_synchronization = False
        if L % self.sparsity_config.block != 0:
            raise ValueError(f"Sequence Length, {L}, needs to be dividable by Block size {self.sparsity_config.block}!")
        nb = L // self.sparsity_config.block
        return self.master_layout[..., :nb, :nb].cpu()

    def _device_layout(self, L, device):
        """uint8 copy of the layout on ``device`` (cached per sequence length: the kernel reads it every call)."""
        cache = self.__dict__.setdefault("_layout_cache", {})
        key = (L, str(device))
        pending = (self._need_layout_synchronization and torch.distributed.is_available()
                   and torch.distributed.is_initialized())  # the first call after init broadcasts rank 0's layout
        if key not in cache or pending:
            cache[key] = self.get_layout(L).to(device=device, dtype=torch.uint8).contiguous()
        return cache[key]

    def transpose_key_for_scores(self, x, L):
        return x  # kept for API parity: no explicit key transpose is needed by this formulation

    def transpose_mask_for_sparse(self, qtype, x, is_key_padding_mask=False):
        x = x.type(qtype)
        if is_key_padding_mask:
            xdim = x.dim()
            for d in range(xdim - 1, 0, -1):
                x = x.squeeze(dim=d)
            return x
        return x.squeeze()

    def forward(self, query, key, value, rpe=None, key_padding_mask=None, attn_mask=None):
        assert query.dtype == key.dtype == value.dtype
        bsz, num_heads, tgt_len, head_dim = query.size()
        if query.shape != key.shape or key.shape != value.shape:
            raise NotImplementedError("only self-attention is supported for now")
        if key_padding_mask is not None:
            key_padding_mask = self.transpose_mask_for_sparse(query.dtype, key_padding_mask, is_key_padding_mask=True)
            key_padding_mask = key_padding_mask.view(bsz, tgt_len)
        if attn_mask is not None:
            attn_mask = self.transpose_mask_for_sparse(query.dtype, attn_mask).view(1, 1, tgt_len, tgt_len)
        if rpe is not None:
            extra = rpe.float().view(1, 1, tgt_len, tgt_len)
            attn_mask = extra if attn_mask is None else (attn_mask.float() if self.attn_mask_mode == "add" else
                                                         (1.0 - attn_mask.float()) * -10000.0) + extra
            mode = "add"
        else:
            mode = self.attn_mask_mode
        layout = self._device_layout(tgt_len, query.device)
        return block_sparse_attention(query, key, value, layout, self.sparsity_config.block, head_dim**-0.5,
                                      key_padding_mask, attn_mask, self.key_padding_mask_mode, mode)
