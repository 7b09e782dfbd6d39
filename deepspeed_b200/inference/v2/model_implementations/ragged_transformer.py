"""One ragged-batch decoder implementation for every supported family.

Role parity: reference ``inference/v2/model_implementations/inference_transformer_base.py`` +
``inference_model_base.py`` + per-family ``model.py`` files, and the module registry under
``inference/v2/modules`` (embedding / pre-norm / attention / linear / moe / unembed / post-norm).

Per layer: ``norm -> packed QKV GEMM -> kv_rotary_append (RoPE + paged KV write) -> attention -> out GEMM ->
[TP all-reduce] -> fused residual+norm -> MLP / MoE -> [TP all-reduce]``.  Prompts that start at position 0 and
are long enough go through the dense flash path (cuDNN SDPA) after their K/V were appended; everything else
(decode, chunked prefill continuation) uses the paged-attention kernel against the blocked cache.
"""
import math
from typing import List, Optional

import os

import torch
import torch.nn.functional as F

from deepspeed_b200 import comm as dist
from deepspeed_b200.ops.kernels import ragged_ops as R
from deepspeed_b200.ops.kernels import transformer_ops as T
from deepspeed_b200.ops.kernels import moe_ops as M
from .arch import ArchSpec

DENSE_PREFILL_MIN = 32
MOE_DENSE_MAX_TOKENS = 64


def _act(x, name):
    if name == "silu":
        return F.silu(x)
    if name == "gelu":
        return F.gelu(x)
    if name == "gelu_new":
        return F.gelu(x, approximate="tanh")
    if name == "relu":
        return F.relu(x)
    raise ValueError(name)


class LayerWeights:
    __slots__ = ("ln1_w", "ln1_b", "ln2_w", "ln2_b", "qkv_w", "qkv_b", "o_w", "o_b", "up_w", "up_b", "down_w", "down_b",
                 "gate_w", "experts_up", "experts_down", "shared_up", "shared_down", "shared_gate")

    def __init__(self):
        for s in self.__slots__:
            setattr(self, s, None)


class RaggedTransformer:
    """Weights are plain tensors (already TP-sharded by ``weights.py``); no nn.Module, no autograd."""

    def __init__(self, spec: ArchSpec, tp_group=None, tp_size=1, tp_rank=0, dtype=torch.bfloat16, device="cuda"):
        self.spec, self.tp_group, self.tp_size, self.tp_rank = spec, tp_group, tp_size, tp_rank
        self.dtype, self.device = dtype, torch.device(device)
        assert spec.heads % tp_size == 0, "query heads must divide the TP degree"
        self.hq = spec.heads // tp_size
        self.hkv = max(1, spec.kv_heads // tp_size)
        self.d = spec.head_dim
        self.embed_w = self.pos_w = self.final_ln_w = self.final_ln_b = self.lm_head_w = self.lm_head_b = None
        self.layers: List[LayerWeights] = [LayerWeights() for _ in range(spec.layers)]
        self.rope = None
        if spec.positional == "rope":
            self.rope = T.RotaryTable(spec.rot_dim, spec.max_positions, base=spec.rope_theta, device=self.device,
                                      scaling=spec.rope_scaling)
        self._state_manager = None
        self.all_logits = False  # v1 `forward` wants every position's logits

    def flat_tensors(self):
        """name -> tensor for every weight this rank holds (quantised weights contribute their codes and scales); the
        contract ``flat_model_helpers`` serialises / restores through."""
        out = {}

        def add(name, v):
            if torch.is_tensor(v):
                out[name] = v
            elif hasattr(v, "q") and hasattr(v, "params"):  # QuantizedWeight
                out[name + ".q"], out[name + ".scales"] = v.q, v.params
            elif isinstance(v, (list, tuple)):
                for i, x in enumerate(v):
                    add(f"{name}.{i}", x)

        for k in ("embed_w", "pos_w", "final_ln_w", "final_ln_b", "lm_head_w", "lm_head_b"):
            add(k, getattr(self, k))
        for i, lw in enumerate(self.layers):
            for sname in lw.__slots__:
                add(f"layers.{i}.{sname}", getattr(lw, sname, None))
        return out

    # ------------------------------------------------------------------ engine-facing API
    def kv_cache_config(self, block_size=128, max_context=8192):
        from ..config_v2 import KVCacheConfig
        name = {torch.bfloat16: "bf16", torch.float16: "fp16", torch.float32: "fp32"}[self.dtype]
        return (KVCacheConfig(block_size=block_size, cache_shape=(self.spec.layers, self.hkv, self.d), cache_dtype=name,
                              max_blocks_per_allocation_group=(max_context + block_size - 1) // block_size), )

    def set_state_manager(self, sm):
        self._state_manager = sm

    def get_kv_requirements(self, seq, max_new_tokens: int, max_new_blocks: int):
        bs = self._state_manager.kv_block_size
        total = seq.seen_tokens + max_new_tokens
        need = (total + bs - 1) // bs - seq.cur_allocated_blocks
        if need <= max_new_blocks:
            return max_new_tokens, max(need, 0)
        cap = (seq.cur_allocated_blocks + max_new_blocks) * bs - seq.seen_tokens
        return max(cap, 0), max_new_blocks

    def get_remaining_block_capacity(self, seq) -> int:
        bs = self._state_manager.kv_block_size
        return (bs - seq.seen_tokens % bs) % bs

    def maybe_allocate_kv(self, seq, n_new_tokens: int) -> None:
        bs = self._state_manager.kv_block_size
        if (seq.seen_tokens + n_new_tokens + bs - 1) // bs <= seq.cur_allocated_blocks:
            return  # fast path (almost every decode step): the current last block still has room
        _, n_blocks = self.get_kv_requirements(seq, n_new_tokens, self._state_manager.free_block_count(0))
        if n_blocks > 0:
            seq.extend_kv_cache(self._state_manager.allocate_blocks(n_blocks))

    def maybe_free_kv(self, seq) -> None:
        pass  # dense (non-sliding-window) caches never free mid-sequence

    # ------------------------------------------------------------------ math
    def _norm(self, x, w, b, residual=None):
        if self.spec.norm == "rms":
            return T.rms_norm(x, w, self.spec.norm_eps, residual=residual)
        return T.layer_norm(x, w, b, self.spec.norm_eps, residual=residual)

    def _reduce(self, x):
        if self.tp_size > 1:
            dist.inference_all_reduce(x, group=self.tp_group)
        return x

    def _linear(self, x, w, b=None):
        from deepspeed_b200.inference.quantization.layers import maybe_quantized_linear
        return maybe_quantized_linear(x, w, b)

    def _attention(self, qkv, cache, batch):
        hq, hkv, d = self.hq, self.hkv, self.d
        bs = self._state_manager.kv_block_size
        R.kv_rotary_append(qkv, cache, self.rope.cos if self.rope else None, self.rope.sin if self.rope else None,
                           batch.seq_of(), batch.pos_of(), batch.block_table(), hq, hkv, d, self.spec.rot_dim, bs)
        layout = batch.seq_layout
        dense = [(t0, n) for (t0, n, seen) in layout if seen == 0 and n >= DENSE_PREFILL_MIN] if qkv.is_cuda else []
        if not dense:
            return R.paged_attention(qkv, cache, batch.seq_of(), batch.pos_of(), batch.block_table(), hq, hkv, d, bs)
        out = torch.empty(qkv.shape[0], hq * d, dtype=qkv.dtype, device=qkv.device)
        covered = 0
        from deepspeed_b200.ops.kernels import attention_sm100 as A
        for t0, n in dense:
            rows = qkv[t0:t0 + n]
            if os.environ.get("DSB200_PREFILL_ATTN", "native") == "native" and A.supports_fwd(rows, hq, hkv, d, 1, n):
                # the in-tree wgmma attention forward, straight on the packed rows (K/V were just rotated in place by
                # kv_rotary_append) and straight into the output rows: no head transposes, any prompt length
                qv, kv_, vv = A.split_packed(rows, hq, hkv)
                A.fwd(qv, kv_, vv, 1, n, hq, hkv, causal=True, out=out[t0:t0 + n], need_lse=False)
                covered += n
                continue
            v3 = rows.view(n, hq + 2 * hkv, d)
            q = v3[:, :hq].transpose(0, 1).unsqueeze(0)
            k = v3[:, hq:hq + hkv].transpose(0, 1).unsqueeze(0)
            v = v3[:, hq + hkv:].transpose(0, 1).unsqueeze(0)
            o = F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=hq != hkv)
            out[t0:t0 + n] = o[0].transpose(0, 1).reshape(n, hq * d)
            covered += n
        if covered < qkv.shape[0]:
            mask = torch.ones(qkv.shape[0], dtype=torch.bool)
            for t0, n in dense:
                mask[t0:t0 + n] = False
            idx = mask.nonzero().squeeze(1).to(qkv.device)
            idx32 = idx.to(torch.int32)
            sub = R.paged_attention(qkv[idx].contiguous(), cache, batch.seq_of()[idx].contiguous(),
                                    batch.pos_of()[idx].contiguous(), batch.block_table(), hq, hkv, d, bs)
            out[idx] = sub
        return out

    def _mlp(self, lw: LayerWeights, x):
        sp = self.spec
        if sp.num_experts:
            return self._moe(lw, x)
        up = self._linear(x, lw.up_w, lw.up_b)
        h = T.gated_act(up, sp.act) if sp.gated_mlp else _act(up, sp.act)
        return self._linear(h, lw.down_w, lw.down_b if self.tp_rank == 0 else None)

    def _moe(self, lw: LayerWeights, x):
        sp = self.spec
        Tn = x.shape[0]
        logits = F.linear(x, lw.gate_w)
        ids, w, counts = M.top_k_gating(logits, sp.top_k, normalize=sp.norm_topk)
        capturing = x.is_cuda and torch.cuda.is_current_stream_capturing()
        if (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_tensor(lw.experts_up) and torch.is_tensor(lw.experts_down)
                and lw.experts_up.dtype == torch.bfloat16 and os.environ.get("DSB200_MOE_GROUPED", "1") != "0"):
            # device-driven grouped GEMM: one persistent wgmma launch per projection streams only the experts that
            # received tokens; offsets never leave the device, so prefill and (graph-captured) decode share this path
            from deepspeed_b200.inference.v2.kernels import moe_gemm
            positions, _, offsets = M.route(ids, sp.num_experts, counts=counts)
            rows = Tn * sp.top_k
            xs, slots = M.scatter(x, ids, positions, offsets, sp.top_k, 0, rows)
            h = T.gated_act(moe_gemm(xs, lw.experts_up, offsets), sp.act)
            ys = moe_gemm(h, lw.experts_down, offsets)
            out = M.gather(ys, w, slots, Tn, sp.top_k)
            return self._moe_shared(lw, x, out)
        if capturing or Tn <= MOE_DENSE_MAX_TOKENS:
            # decode-sized batch: every expert's weights get streamed once anyway (weight-bandwidth bound), so run
            # all experts on all rows and mask — no host sync, static shapes, CUDA-graph capturable.
            out = torch.zeros(Tn, x.shape[1], dtype=torch.float32, device=x.device)
            for e in range(sp.num_experts):
                we = (w * (ids == e)).sum(-1, keepdim=True)
                ye = F.linear(T.gated_act(F.linear(x, lw.experts_up[e]), sp.act), lw.experts_down[e])
                out.addcmul_(ye.float(), we)
            out = out.to(x.dtype)
            return self._moe_shared(lw, x, out)
        positions, counts2, offsets = M.route(ids, sp.num_experts)
        rows = Tn * sp.top_k
        xs, slots = M.scatter(x, ids, positions, offsets, sp.top_k, 0, rows)
        off = offsets.tolist()
        ys = torch.empty(rows, x.shape[1], dtype=x.dtype, device=x.device)
        for e in range(sp.num_experts):
            s, t = off[e], off[e + 1]
            if t > s:
                h = T.gated_act(F.linear(xs[s:t], lw.experts_up[e]), sp.act)
                ys[s:t] = F.linear(h, lw.experts_down[e])
        out = M.gather(ys, w, slots, Tn, sp.top_k)
        return self._moe_shared(lw, x, out)

    def _moe_shared(self, lw, x, out):
        sp = self.spec
        if lw.shared_up is not None:
            sh = F.linear(T.gated_act(F.linear(x, lw.shared_up), sp.act), lw.shared_down)
            if lw.shared_gate is not None:
                sh = sh * torch.sigmoid(F.linear(x, lw.shared_gate))
            out = out + sh
        return out

    @torch.no_grad()
    def forward(self, batch) -> torch.Tensor:
        sp = self.spec
        ids = batch.input_ids()
        h = R.ragged_embed(ids, self.embed_w, batch.pos_of() if self.pos_w is not None else None, self.pos_w, sp.pos_offset)
        residual = h
        x = self._norm(residual, self.layers[0].ln1_w, self.layers[0].ln1_b)
        for i, lw in enumerate(self.layers):
            cache = self._state_manager.get_cache(i)
            qkv = self._linear(x, lw.qkv_w, lw.qkv_b)
            att = self._attention(qkv, cache, batch)
            a = self._reduce(self._linear(att, lw.o_w, lw.o_b if self.tp_rank == 0 else None))
            if sp.parallel_residual:
                xm = x if sp.shared_ln else self._norm(residual, lw.ln2_w, lw.ln2_b)
                m = self._reduce(self._mlp(lw, xm))
                residual = residual + a + m
                nxt = self.layers[i + 1] if i + 1 < sp.layers else None
                x = self._norm(residual, nxt.ln1_w, nxt.ln1_b) if nxt is not None else residual
            else:
                x, residual = self._norm(a, lw.ln2_w, lw.ln2_b, residual=residual)
                m = self._reduce(self._mlp(lw, x))
                nxt = self.layers[i + 1] if i + 1 < sp.layers else None
                if nxt is not None:
                    x, residual = self._norm(m, nxt.ln1_w, nxt.ln1_b, residual=residual)
                else:
                    residual = residual + m
        last = residual if self.all_logits else R.row_gather(residual, batch.last_token_index())
        if sp.final_norm:
            last = self._norm(last, self.final_ln_w, self.final_ln_b)
        logits = F.linear(last, self.lm_head_w, self.lm_head_b)
        if self.tp_size > 1 and getattr(self, "lm_head_sharded", False):
            parts = [torch.empty_like(logits) for _ in range(self.tp_size)]
            dist.all_gather(parts, logits, group=self.tp_group)
            logits = torch.cat(parts, dim=-1)
        return logits
