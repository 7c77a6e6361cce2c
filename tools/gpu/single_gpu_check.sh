#!/bin/bash
# Everything measured on ONE H100, in the order the driver runs it plus the profiling passes.  Run from the repo root
# (about 6 minutes); outputs land in the directory created below.
mkdir -p gpurun_out
timeout 1200 python -m pytest tests -x -q -m gpu 2>&1 | tail -4 | tee gpurun_out/pytest_gpu.log
timeout 200 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
timeout 600 python bench.py > gpurun_out/bench.json 2> gpurun_out/bench.err
echo "stdout lines: $(wc -l < gpurun_out/bench.json)"; cut -c1-400 gpurun_out/bench.json
timeout 300 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/bench_reference.json 2>/dev/null; cut -c1-300 gpurun_out/bench_reference.json
timeout 300 python tools/sweep.py > gpurun_out/sweep.jsonl 2> gpurun_out/sweep.err
NCU=1 bash tools/gpu/ab_check.sh
bash tools/gpu/dropin_timing.sh
bash tools/gpu/sanitize.sh
ls -la gpurun_out
