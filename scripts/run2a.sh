#!/bin/bash
# GPU run 2a (1 GPU): dSwiGLU epilogue v2, full tuning table, two-phase (clip / GAS) arms at Llama-3-8B scale
mkdir -p gpurun_out; rm -f gpurun_out/r2a_status.txt
timeout 600 python -m pytest tests/gpu/test_gemm_gpu.py -x -q > gpurun_out/r2a_gemm_tests.log 2>&1
echo "gemm tests rc=$?" >> gpurun_out/r2a_status.txt
timeout 900 python scripts/tune_gemm.py --models llama3-8b,phi3-mini --group-m 0,4,8,16 --out gpurun_out/gemm_table.json --report gpurun_out/gemm_tune_report.json > gpurun_out/r2a_tune.log 2>&1
echo "tune rc=$?" >> gpurun_out/r2a_status.txt
cp gpurun_out/gemm_table.json deepspeed_b200/ops/gemm_table.json 2>/dev/null
timeout 600 python bench.py --gpus 1 --steps 8 --warmup 3 > gpurun_out/r2a_bench_n1.json 2> gpurun_out/r2a_bench_n1.err
echo "bench rc=$?" >> gpurun_out/r2a_status.txt
timeout 600 python bench.py --gpus 1 --steps 6 --warmup 3 --clip 1.0 > gpurun_out/r2a_bench_n1_clip.json 2> gpurun_out/r2a_bench_n1_clip.err
echo "bench clip rc=$?" >> gpurun_out/r2a_status.txt
timeout 600 python bench.py --gpus 1 --steps 3 --warmup 3 --gas 4 > gpurun_out/r2a_bench_n1_gas4.json 2> gpurun_out/r2a_bench_n1_gas4.err
echo "bench gas rc=$?" >> gpurun_out/r2a_status.txt
timeout 600 python -m pytest tests/gpu -x -q -m gpu --deselect tests/gpu/test_gemm_gpu.py > gpurun_out/r2a_gpu_tests.log 2>&1
echo "gpu tests rc=$?" >> gpurun_out/r2a_status.txt
tail -3 gpurun_out/r2a_gemm_tests.log; grep -E "dswiglu|wrote" gpurun_out/r2a_tune.log; for f in gpurun_out/r2a_bench_n1*.json; do python - "$f" <<'PY'
import json,sys
try:
    d=json.loads(open(sys.argv[1]).read().strip().splitlines()[-1]); print(sys.argv[1], d["value"], d["ms_per_step"], d["e2e"]["value"], d["details"]["gemm_choices"]["own_wgmma"], d["details"]["gemm_choices"]["cublas_shapes"], d["details"]["fused_in_backward_optimizer"])
except Exception as e: print(sys.argv[1], "ERR", e)
PY
done; tail -3 gpurun_out/r2a_gpu_tests.log; cat gpurun_out/r2a_status.txt
