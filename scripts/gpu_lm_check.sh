#!/bin/bash
# LM-side check after a kernel change: LM GPU tests, codec attention tests, the LM decode bench leg only
mkdir -p gpurun_out
timeout 900 python -m pytest tests/test_lm_gpu.py -x -q -rA 2>&1 | tail -60 > gpurun_out/r2_lm_tests.log; tail -4 gpurun_out/r2_lm_tests.log
timeout 300 python -m pytest tests/test_codec_gpu.py tests/test_codec_round2_gpu.py -x -q -k "attention or streaming or reset or cfg2" 2>&1 | tail -5
timeout 600 python - <<'PY' 2>&1 | tail -30
import json, sys, torch
sys.path.insert(0, '.')
import bench
dev = torch.device('cuda', 0)
r = bench.lm_decode_bench(dev, steps=10, warmup=3)
r.pop('gemm_by_shape_NK', None)
print(json.dumps(r, indent=1))
json.dump(r, open('gpurun_out/r2_lm_decode.json', 'w'), indent=1)
PY
