#!/bin/bash
# Run from the repository root on an H100:  bash scripts/gpu_checks.sh [quick]
# Parity tests, smoke, bench (+ reference arm), ncu launch list and --set full captures, secondary configs.
set -u
mkdir -p gpurun_out
cd "${GRAFT_REPO_ROOT:-.}"
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw --format=csv > gpurun_out/gpu.txt 2>&1
nproc > gpurun_out/nproc.txt; lscpu | grep 'Model name' >> gpurun_out/nproc.txt

echo "== pytest -m gpu"; timeout 1500 python -m pytest tests -m gpu -q > gpurun_out/pytest_gpu_full.log 2>&1; tail -25 gpurun_out/pytest_gpu_full.log | tee gpurun_out/pytest_gpu.log
echo "== smoke"; timeout 300 python -c 'import __graft_entry__ as g; g.smoke()' 2>&1 | tail -5 | tee gpurun_out/smoke.log

echo "== bench"; timeout 600 python bench.py 2> gpurun_out/bench.err | tee gpurun_out/bench.json | cut -c1-400
tail -3 gpurun_out/bench.err
echo "== reference arm"; timeout 400 python bench.py --impl reference --steps 20 --warmup 3 2>> gpurun_out/bench.err | tee gpurun_out/bench_reference.json | cut -c1-300
if [ "${1:-}" = "quick" ]; then exit 0; fi

echo "== other configs"; timeout 600 python scripts/bench_configs.py 2> gpurun_out/configs.err | tee gpurun_out/bench_configs.json | cut -c1-300
echo "== train step profile"; timeout 600 python scripts/profile_train_step.py 2> gpurun_out/train.err | tee gpurun_out/train_step_profile.json | cut -c1-600

echo "== ncu launch list (bench.py)"
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/launches.csv \
    python bench.py --steps 48 --warmup 3 --no-cpu-baseline --no-e2e > gpurun_out/bench_under_ncu.log 2>&1
echo "== ncu launch list (other configs: rnea + backward kernels)"
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:'rnea|fk_jacobian|reduce_partials' -c 200 --csv \
    --log-file gpurun_out/launches_configs.csv python scripts/profile_train_step.py > gpurun_out/train_under_ncu.log 2>&1
echo "== ncu --set full (fk_jacobian, batch 65536 and 2^22)"
timeout 900 ncu --set full --clock-control none --import-source on -k regex:fk_jacobian -s 20 -c 3 -f -o gpurun_out/fk_small \
    python bench.py --steps 48 --warmup 3 --no-cpu-baseline --no-e2e --no-large > gpurun_out/ncu_small.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:fk_jacobian -s 105 -c 2 -f -o gpurun_out/fk_large \
    python bench.py --steps 48 --warmup 3 --no-cpu-baseline --no-e2e > gpurun_out/ncu_large.log 2>&1
echo "== ncu --set full (rnea forward + backward)"
timeout 900 ncu --set full --clock-control none --import-source on -k regex:rnea -s 12 -c 4 -f -o gpurun_out/rnea \
    python scripts/profile_train_step.py > gpurun_out/ncu_rnea.log 2>&1
ls -la gpurun_out
