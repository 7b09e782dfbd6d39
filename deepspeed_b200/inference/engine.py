"""Inference engine (v1 API).  Reference: ``inference/engine.py:39 InferenceEngine``.

Three ways to serve, chosen by config exactly like the reference:

* ``replace_with_kernel_inject=True`` — the module's weights are re-packed into the ragged fused-kernel model
  (``inference/v2/model_implementations``) with a paged KV cache; ``forward`` / ``generate`` run on it.  The
  reference swaps each HF block for ``DeepSpeedTransformerInference``; here the whole decoder stack is one
  implementation shared with the v2 engine, so v1 users get the same kernels and CUDA-graphed decode.
* ``tensor_parallel.tp_size > 1`` without injection — AutoTP shards the module's linears in place.
* otherwise — dtype conversion (+ optional CUDA-graph replay of the module's static-shape forward).
"""
import os
import time
from typing import Optional

import torch
from torch import nn

from deepspeed_b200 import comm as dist
from deepspeed_b200.accelerator import get_accelerator
from deepspeed_b200.utils import groups
from deepspeed_b200.utils.logging import log_dist, logger
from .config import DeepSpeedInferenceConfig


class _Output(dict):
    """Minimal CausalLM output: attribute + tuple + dict access."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __iter__(self):
        return iter(self.values())

    def __getitem__(self, k):
        if isinstance(k, int):
            return list(self.values())[k]
        return super().__getitem__(k)


class InferenceEngine(nn.Module):
    inference_mp_group = None
    inference_ep_group = None
    expert_mp_group = None

    def __init__(self, model, config: DeepSpeedInferenceConfig):
        super().__init__()
        self._config = config
        self.module = model
        self.dtype = config.dtype
        self.mp_world_size = config.tensor_parallel.tp_size
        self.mpu = config.tensor_parallel.mpu
        self.injection_dict = config.injection_policy
        self.cuda_graph_created = False
        self._cuda_graphs = None
        self._ragged = None
        self._model_times = []
        self.model_profile_enabled = False
        self._uid = 0
        self.checkpoint_engine = None

        if self.mp_world_size > 1 or config.moe and getattr(config.moe, "ep_size", 1) > 1:
            if not dist.is_initialized():
                dist.init_distributed()
        self._create_model_parallel_group(config)
        dev = get_accelerator().current_device_name() if get_accelerator().is_available() else "cpu"
        self.device = torch.device(dev)

        if config.checkpoint is not None and not config.replace_with_kernel_inject:
            self._load_checkpoint(config.checkpoint)

        if config.replace_with_kernel_inject:
            self._inject_kernels()
        else:
            if self.dtype in (torch.float16, torch.bfloat16, torch.float32) and not config.keep_module_on_host:
                self.module.to(self.dtype)
            if self.mp_world_size > 1 and config.tensor_parallel.enabled:
                from deepspeed_b200.module_inject.auto_tp import AutoTP
                AutoTP(self.module, mp_group=self.mp_group, mp_size=self.mp_world_size,
                       all_reduce_linears=_policy_names(self.injection_dict)).replace()
            if not config.keep_module_on_host:
                self.module.to(self.device)
            if config.quant.enabled and config.quant.weight.post_init_quant:
                from .quantization import _init_group_wise_weight_quantization
                _init_group_wise_weight_quantization(self.module, {"weight_quantization": {
                    "post_init_quant": config.quant.weight.post_init_quant}})
        if config.save_mp_checkpoint_path:
            self._save_mp_checkpoint(config.save_mp_checkpoint_path)
        self.module.eval()
        self.local_cuda_graph = False

    # ------------------------------------------------------------------ setup
    def _create_model_parallel_group(self, config):
        self.mp_group = None
        if config.tensor_parallel.tp_group is not None:
            self.mp_group = config.tensor_parallel.tp_group
        elif self.mpu is not None:
            self.mp_group = self.mpu.get_model_parallel_group()
        elif self.mp_world_size > 1:
            if InferenceEngine.inference_mp_group is None:
                if groups.ranks_of("tp") is None:
                    groups._init_tp_mesh_device(tensor_model_parallel_size=self.mp_world_size)
                InferenceEngine.inference_mp_group = groups.get_tensor_model_parallel_group()
            self.mp_group = InferenceEngine.inference_mp_group

    def _inject_kernels(self):
        from .v2.config_v2 import RaggedInferenceEngineConfig
        from .v2.engine_v2 import InferenceEngineV2
        from .v2.model_implementations import RaggedTransformer, arch_from_hf_config, load_hf_weights, weights_from_b200_model
        cfg = self._config
        max_ctx = max(cfg.max_out_tokens, 64)
        ec = RaggedInferenceEngineConfig(state_manager={"max_context": max_ctx, "max_ragged_batch_size":
                                                        max(4 * max_ctx, 2048), "max_ragged_sequence_count": 256},
                                         cuda_graph_decode=cfg.enable_cuda_graph)
        # v1 API serves at most 256 concurrent sequences of max_out_tokens: size the KV pool for exactly that instead
        # of claiming all free HBM (the v2 factory default)
        ec.state_manager.memory_config.mode = "allocate"
        ec.state_manager.memory_config.size = 64 if self.device.type != "cuda" else max(64, 256 * ((max_ctx + 127) // 128))
        rank = dist.get_rank(self.mp_group) if self.mp_group is not None else 0
        quant = "int8" if self.dtype == torch.int8 else None
        dtype = torch.float16 if self.dtype == torch.int8 else self.dtype
        hf_cfg = getattr(self.module, "config", None)
        from .v2.model_implementations.arch import SUPPORTED_MODEL_TYPES
        layerwise = os.environ.get("DSB200_LAYERWISE_INJECTION", "0") == "1"
        if hf_cfg is not None and hasattr(hf_cfg, "model_type") and (hf_cfg.model_type not in SUPPORTED_MODEL_TYPES or layerwise):
            # encoders (BERT, DistilBERT, RoBERTa, CLIP), BLOOM / GPT-Neo and anything else the ragged engine has no
            # architecture entry for: per-layer fused kernels through the policy / container registry, the rest of the
            # Hugging Face model (embeddings, pooler, heads, generate loop) stays as is
            from deepspeed_b200.module_inject.replace_module import replace_transformer_layer
            sd = None
            if isinstance(cfg.checkpoint, str) and os.path.isdir(cfg.checkpoint):
                from .v2.engine_factory import HuggingFaceCheckpointEngine
                eng = HuggingFaceCheckpointEngine(cfg.checkpoint)
                sd = dict(eng.parameters())
            self.module.to(dtype)
            replace_transformer_layer(None, self.module, checkpoint_dict=sd, config=cfg)
            self.module.to(self.device)
            return
        if hf_cfg is not None and hasattr(hf_cfg, "model_type"):
            spec = arch_from_hf_config(hf_cfg)
            model = RaggedTransformer(spec, self.mp_group, self.mp_world_size, rank, dtype, self.device)
            if isinstance(cfg.checkpoint, str) and os.path.isdir(cfg.checkpoint):
                from .v2.engine_factory import HuggingFaceCheckpointEngine
                load_hf_weights(model, HuggingFaceCheckpointEngine(cfg.checkpoint).get, quant)
            else:
                load_hf_weights(model, self.module.state_dict().get, quant)
        else:
            from .v2.engine_factory import build_engine_from_model
            ec.tensor_parallel.tp_size = self.mp_world_size
            self._ragged = build_engine_from_model(self.module, ec, dtype=dtype, device=self.device)
            return
        self._ragged = InferenceEngineV2(model, ec, tp_group=self.mp_group)

    def _load_checkpoint(self, ckpt):
        """``ckpt``: path to a state-dict file, a dir of shards, or the reference's json descriptor
        ``{"type": .., "checkpoints": [...], "version": ..}``."""
        import json
        if isinstance(ckpt, str) and ckpt.endswith(".json"):
            with open(ckpt) as f:
                ckpt = json.load(f)
        files = []
        if isinstance(ckpt, dict):
            base = ckpt.get("base_dir", self._config.base_dir or "")
            files = [os.path.join(base, c) for c in ckpt.get("checkpoints", [])]
        elif os.path.isdir(ckpt):
            files = sorted(os.path.join(ckpt, f) for f in os.listdir(ckpt) if f.endswith((".pt", ".bin")))
        else:
            files = [ckpt]
        sd = {}
        for f in files:
            part = torch.load(f, map_location="cpu", weights_only=False)
            sd.update(part.get("module", part.get("model", part)) if isinstance(part, dict) else part)
        missing, unexpected = self.module.load_state_dict(sd, strict=False)
        if missing:
            logger.warning(f"inference checkpoint: {len(missing)} missing keys (first: {missing[:3]})")

    def _save_mp_checkpoint(self, path):
        os.makedirs(path, exist_ok=True)
        rank = dist.get_rank(self.mp_group) if self.mp_group is not None else 0
        if self._ragged is not None:
            self._ragged.serialize(path)
        else:
            torch.save(self.module.state_dict(), os.path.join(path, f"tp_{rank:02d}.pt"))
        if rank == 0:
            import json
            with open(os.path.join(path, "ds_inference_config.json"), "w") as f:
                json.dump({"type": "ds_model", "version": 1.0, "tp_size": self.mp_world_size,
                           "checkpoints": [f"tp_{r:02d}.pt" for r in range(self.mp_world_size)]}, f)

    # ------------------------------------------------------------------ profiling
    def profile_model_time(self, use_cuda_events=True):
        self.model_profile_enabled = True
        self.use_cuda_events = use_cuda_events and torch.cuda.is_available()

    def model_times(self):
        t, self._model_times = self._model_times, []
        return t

    # ------------------------------------------------------------------ forward / generate
    def _next_uids(self, n):
        u = list(range(self._uid, self._uid + n))
        self._uid += n
        return u

    def _ragged_forward(self, input_ids, attention_mask=None):
        B, S = input_ids.shape
        lens = attention_mask.sum(1).tolist() if attention_mask is not None else [S] * B
        uids = self._next_uids(B)
        seqs = [input_ids[b, S - lens[b]:] if attention_mask is not None and attention_mask[b, 0] == 0 else
                input_ids[b, :lens[b]] for b in range(B)]
        self._ragged._batch.clear()
        logits = self._ragged_put_all(uids, seqs)
        for u in uids:
            self._ragged.flush(u)
        out = torch.zeros(B, S, logits.shape[-1], dtype=logits.dtype, device=logits.device)
        t = 0
        for b in range(B):
            n = lens[b]
            if attention_mask is not None and attention_mask[b, 0] == 0:
                out[b, S - n:] = logits[t:t + n]
            else:
                out[b, :n] = logits[t:t + n]
            t += n
        return out

    def _ragged_put_all(self, uids, seqs):
        m = self._ragged.model
        m.all_logits = True
        try:
            return self._ragged.put(uids, [s.cpu() for s in seqs])
        finally:
            m.all_logits = False

    def forward(self, *inputs, **kwargs):
        start = None
        if self.model_profile_enabled:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            start = time.time()
        if self._ragged is not None:
            input_ids = kwargs.get("input_ids", inputs[0] if inputs else None)
            logits = self._ragged_forward(input_ids, kwargs.get("attention_mask"))
            out = _Output(logits=logits)
            out = (logits, ) if kwargs.get("return_dict") is False else out
        elif self._config.enable_cuda_graph and torch.cuda.is_available():
            out = self._graph_forward(*inputs, **kwargs)
        else:
            with torch.no_grad():
                out = self.module(*inputs, **kwargs)
        if start is not None:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            self._model_times.append((time.time() - start) * 1e3)
        return out

    def _graph_forward(self, *inputs, **kwargs):
        key = tuple((tuple(t.shape), t.dtype) for t in list(inputs) + list(kwargs.values()) if torch.is_tensor(t))
        if self._cuda_graphs is None:
            self._cuda_graphs = {}
        ent = self._cuda_graphs.get(key)
        if ent is None:
            s_in = [t.clone() if torch.is_tensor(t) else t for t in inputs]
            s_kw = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in kwargs.items()}
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s), torch.no_grad():
                for _ in range(3):
                    self.module(*s_in, **s_kw)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g), torch.no_grad():
                s_out = self.module(*s_in, **s_kw)
            ent = self._cuda_graphs[key] = (g, s_in, s_kw, s_out)
            self.cuda_graph_created = True
        g, s_in, s_kw, s_out = ent
        for d, srct in zip(s_in, inputs):
            if torch.is_tensor(d):
                d.copy_(srct)
        for k, v in kwargs.items():
            if torch.is_tensor(v):
                s_kw[k].copy_(v)
        g.replay()
        return s_out

    @torch.no_grad()
    def generate(self, *inputs, **kwargs):
        if self._ragged is None:
            if "num_beams" in kwargs and kwargs["num_beams"] > 1 and self._config.replace_with_kernel_inject:
                raise NotImplementedError("beam search is not supported with kernel injection")
            return self.module.generate(*inputs, **kwargs)
        input_ids = kwargs.pop("input_ids", inputs[0] if inputs else None)
        eos_default = getattr(getattr(self.module, "config", None), "eos_token_id", None)
        out, self._uid = ragged_generate(self._ragged, input_ids, self._uid, self._config.max_out_tokens,
                                         eos_default=eos_default, **kwargs)
        return out

    def destroy(self):
        self._ragged = None
        self._cuda_graphs = None
        InferenceEngine.inference_mp_group = None

    # ---- model-specific patches of the AutoTP path (reference ``inference/engine.py:207-228``) ---------------------------
    def remove_mask_prepare_for_bloom(self):
        """BLOOM builds its own causal mask; the fused layers want the raw padding mask."""
        tr = getattr(self.module, "transformer", None)
        if tr is not None and hasattr(tr, "_prepare_attn_mask"):
            tr._prepare_attn_mask = lambda attention_mask, *args, **kwargs: attention_mask

    def build_alibi_tensor(self):
        """Under tensor parallelism ALiBi slopes must be generated for this rank's heads only."""
        from deepspeed_b200.module_inject import auto_tp_model_utils as U
        tr = getattr(self.module, "transformer", None)
        if tr is not None:
            if hasattr(tr, "build_alibi_tensor"):
                tr.build_alibi_tensor = U.build_bloom_alibi_tensor
            if hasattr(tr, "build_mpt_alibi_tensor"):
                tr.build_mpt_alibi_tensor_orig = tr.build_mpt_alibi_tensor
                tr.__class__.build_mpt_alibi_tensor = U.build_mpt_alibi_tensor
        inner = getattr(self.module, "model", None)
        if inner is not None and hasattr(inner, "get_alibi_mask"):
            inner.get_alibi_mask_orig = inner.get_alibi_mask
            inner.__class__.get_alibi_mask = U.get_alibi_mask

    def build_attn_bias(self):
        from deepspeed_b200.module_inject import auto_tp_model_utils as U
        tr = getattr(self.module, "transformer", None)
        if tr is not None and hasattr(tr, "_attn_bias"):
            tr._attn_bias_orig = tr._attn_bias
            tr.__class__._attn_bias = U.build_mpt_atten_bias_tensor

    def load_model_with_checkpoint(self, r_module):
        """Fill a (possibly meta-initialised) module tree from ``self.sd`` -- the state dict of the checkpoint shard being
        loaded -- slicing tensors for this TP rank; embeddings tied to ``lm_head`` are re-tied afterwards."""
        from deepspeed_b200.module_inject.auto_tp import Loading
        sd = getattr(self, "sd", None)
        assert sd is not None, "set engine.sd (the checkpoint state dict) before load_model_with_checkpoint"

        def walk(mod, prefix=""):
            for name, child in mod.named_children():
                full = prefix + name + "."
                if Loading.is_load_module(child) and any(k.startswith(full) for k in sd):
                    Loading.load(child, sd, full, mp_group=self.mp_group)
                    Loading.load_buffer(child, sd, full)
                else:
                    walk(child, full)

        walk(r_module)
        emb, head = None, getattr(r_module, "lm_head", None)
        for n, m in r_module.named_modules():
            if isinstance(m, nn.Embedding) and ("embed_tokens" in n or "wte" in n or "word_embeddings" in n):
                emb = m
        if emb is not None and head is not None and getattr(head, "weight", None) is not None and head.weight.is_meta:
            head.weight = emb.weight

    @property
    def is_compiled(self) -> bool:
        return bool(getattr(self, "_is_compiled", False))


@torch.no_grad()
def ragged_generate(ragged, input_ids, uid0, max_out_tokens, eos_default=None, **kwargs):
    """Greedy / sampling generation on a ragged engine; returns (tokens [B, S+new], next free uid)."""
    if kwargs.get("num_beams", 1) > 1:
        raise NotImplementedError("DeepSpeed-H100 kernel-injected generate supports greedy / sampling only")
    max_new = kwargs.get("max_new_tokens")
    if max_new is None:
        max_new = kwargs.get("max_length", input_ids.shape[1] + 20) - input_ids.shape[1]
    if input_ids.shape[1] + max_new > max_out_tokens:
        raise RuntimeError(f"Input with size {input_ids.shape[1]} + {max_new} new tokens exceeds max_out_tokens "
                           f"{max_out_tokens}; raise `max_tokens` in the inference config")
    do_sample = kwargs.get("do_sample", False)
    temperature, top_k, top_p = kwargs.get("temperature", 1.0), kwargs.get("top_k", 0), kwargs.get("top_p", 1.0)
    eos = kwargs.get("eos_token_id", eos_default)
    eos = set(eos) if isinstance(eos, (list, tuple)) else ({eos} if eos is not None else set())
    pad = kwargs.get("pad_token_id", next(iter(eos)) if eos else 0)
    B = input_ids.shape[0]
    mask = kwargs.get("attention_mask")
    uids = list(range(uid0, uid0 + B))
    seqs = [input_ids[b][mask[b].bool()] if mask is not None else input_ids[b] for b in range(B)]
    logits = ragged.put(uids, [s.cpu() for s in seqs])
    done = [False] * B
    new_tokens = [[] for _ in range(B)]
    for step in range(max_new):
        nxt = _sample(logits, do_sample, temperature, top_k, top_p)
        live_u, live_t = [], []
        nxt_host = nxt.tolist()
        k = 0
        for b in range(B):
            if done[b]:
                continue
            tok = nxt_host[k]
            k += 1
            new_tokens[b].append(tok)
            if tok in eos:
                done[b] = True
            else:
                live_u.append(uids[b])
                live_t.append(torch.tensor([tok]))
        if not live_u or step == max_new - 1:
            break
        logits = ragged.put(live_u, live_t)
    for u in uids:
        ragged.flush(u)
    L = max(len(t) for t in new_tokens)
    out = torch.full((B, input_ids.shape[1] + L), pad, dtype=input_ids.dtype, device=input_ids.device)
    out[:, :input_ids.shape[1]] = input_ids
    for b in range(B):
        out[b, input_ids.shape[1]:input_ids.shape[1] + len(new_tokens[b])] = torch.tensor(new_tokens[b],
                                                                                         dtype=input_ids.dtype)
    return out, uid0 + B



def _policy_names(injection_dict):
    names = []
    for v in (injection_dict or {}).values():
        names.extend(n.split(".")[-1] for n in (v if isinstance(v, (tuple, list)) else (v, )))
    return names


def _sample(logits, do_sample, temperature, top_k, top_p):
    if not do_sample:
        return logits.argmax(-1)
    logits = logits.float() / max(temperature, 1e-5)
    if top_k:
        kth = logits.topk(top_k, dim=-1).values[:, -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if top_p < 1.0:
        sl, si = logits.sort(dim=-1, descending=True)
        cp = sl.softmax(-1).cumsum(-1)
        cut = cp - sl.softmax(-1) > top_p
        sl = sl.masked_fill(cut, float("-inf"))
        logits = torch.full_like(logits, float("-inf")).scatter(-1, si, sl)
    return torch.multinomial(logits.softmax(-1), 1).squeeze(-1)
