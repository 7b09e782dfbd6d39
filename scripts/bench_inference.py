"""Ragged-engine serving microbenchmark: prefill + CUDA-graphed decode throughput on one H100.
python scripts/bench_inference.py [--model llama3-8b] [--batch 64] [--prompt 512] [--new 64]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepspeed_b200.inference.v2 import build_engine_from_model
from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
from deepspeed_b200.utils import OnDevice

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="llama3-8b")
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--prompt", type=int, default=512)
ap.add_argument("--new", type=int, default=64)
ap.add_argument("--layers", type=int, default=0)
a = ap.parse_args()
cfg = llama_config(a.model, **({"num_hidden_layers": a.layers} if a.layers else {}))
torch.manual_seed(0)
with torch.device("cuda"):
    model = LlamaForCausalLM(cfg).to(torch.bfloat16)
eng = build_engine_from_model(model, {"state_manager": {"max_context": a.prompt + a.new + 8, "max_ragged_batch_size":
                                                        max(a.batch, 8192), "max_ragged_sequence_count": max(a.batch, 8),
                                                        "memory_config": {"mode": "reserve", "size": 8_000_000_000}}})
del model
torch.cuda.empty_cache()
# warm-up: cuBLAS heuristics, cuDNN SDPA plan, first-touch of the KV pool
eng.put([10**6], [torch.randint(0, cfg.vocab_size, (a.prompt, ))])
eng.put([10**6], [torch.randint(0, cfg.vocab_size, (1, ))])
eng.flush(10**6)
torch.cuda.synchronize()
uids = list(range(a.batch))
prompts = [torch.randint(0, cfg.vocab_size, (a.prompt, )) for _ in uids]
# prefill in ragged batches of <= 8192 tokens
per = max(1, 8192 // a.prompt)
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize()
s.record()
logits = []
for i in range(0, a.batch, per):
    logits.append(eng.put(uids[i:i + per], prompts[i:i + per]))
e.record()
torch.cuda.synchronize()
prefill_ms = s.elapsed_time(e)
nxt = torch.cat(logits).argmax(-1).cpu()
# warm decode (captures the CUDA graph), then time
for _ in range(3):
    lg = eng.put(uids, [t.reshape(1) for t in nxt])
    nxt = lg.argmax(-1).cpu()
torch.cuda.synchronize()
s.record()
for _ in range(a.new):
    lg = eng.put(uids, [t.reshape(1) for t in nxt])
    nxt = lg.argmax(-1).cpu()
e.record()
torch.cuda.synchronize()
dec_ms = s.elapsed_time(e)
weights_gb = cfg.num_parameters() * 2 / 1e9
print(json.dumps({"model": a.model, "batch": a.batch, "prompt": a.prompt, "new_tokens": a.new,
                  "prefill_tokens_per_s": a.batch * a.prompt / prefill_ms * 1e3, "prefill_ms": prefill_ms,
                  "decode_tokens_per_s": a.batch * a.new / dec_ms * 1e3, "decode_ms_per_step": dec_ms / a.new,
                  "weight_stream_GBps_at_decode": weights_gb / (dec_ms / a.new / 1e3),
                  "max_mem_gb": torch.cuda.max_memory_allocated() / 2**30}))
