#!/bin/bash
# round 2, call G: balanced tracker partition, bilateral interior path, merged pyramids: parity + bench
mkdir -p gpurun_out
echo "== parity + ref pins"; timeout 1200 python -m pytest tests/test_gpu_parity.py tests/test_gpu_ref.py tests/test_gpu_seg.py -q -m gpu -p no:cacheprovider --timeout 900 --tb=short > gpurun_out/pytest_parity_g.log 2>&1; echo rc=$?; tail -n 12 gpurun_out/pytest_parity_g.log | cut -c1-400
echo "== bench main line"; MFB200_BENCH_LEGS=0 timeout 400 python bench.py --steps 100 --warmup 10 > gpurun_out/bench_g.json 2> gpurun_out/bench_g.err; echo rc=$?; python -c "
import json; b=json.load(open('gpurun_out/bench_g.json')); print(b['value'], b['e2e']['value'], {k:v['avg_ms'] for k,v in b['roofline']['kernels'].items()})"; tail -n 3 gpurun_out/bench_g.err
echo "== track timing"; MFB200_TAG=timing timeout 300 python scripts/track_timing.py > gpurun_out/track_timing_g.json 2> gpurun_out/track_timing_g.err; echo rc=$?; head -c 2500 gpurun_out/track_timing_g.json | tr -d '\n '; echo; tail -n 3 gpurun_out/track_timing_g.err
