#!/bin/bash
# Validation on one H100 (run from the repo root): the GPU test suite, smoke(), both bench arms.
# Profiles are tools/profile_r02.sh, sanitizer runs tools/sanitize.sh. Outputs -> gpurun_out/.
mkdir -p gpurun_out
timeout 900 python -m pytest tests -x -q -m gpu --timeout 300 > gpurun_out/final_tests.log 2>&1; tail -n 3 gpurun_out/final_tests.log
timeout 120 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" > gpurun_out/final_smoke.log 2>&1; tail -n 1 gpurun_out/final_smoke.log
timeout 300 python bench.py --impl reference --steps 10 --warmup 2 > gpurun_out/final_ref.log 2>&1
timeout 400 python bench.py > gpurun_out/final_ours.log 2>&1
grep -c "^{" gpurun_out/final_ref.log gpurun_out/final_ours.log
python tools/round_probe.py 22 2 > gpurun_out/final_probe.txt 2>&1; tail -n 3 gpurun_out/final_probe.txt
