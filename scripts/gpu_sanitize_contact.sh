#!/bin/bash
# bash scripts/gpu_sanitize_contact.sh : compute-sanitizer memcheck / racecheck over the contact adjoint (csrc/contact_backward.cu)
# at small batches: the rung cases of tests/test_contact_backward_coverage_gpu.py (70-196 rows; not the persistent-loop
# cases of 10^4-10^5 rows) and the fp64-oracle cases of tests/test_contact_backward_gpu.py (48 rows).  Observation only:
# one pass of each, every step under a timeout.
set -u
cd "$(dirname "$0")/.."                             # the repository root
OUT=${OUT:-$(mktemp -d -t contact_sanitize.XXXXXX)}  # where the sanitizer logs go
mkdir -p "$OUT"
echo "logs in $OUT"
RUNGS="every_rung or null_outputs or unsolved"
for tool in memcheck racecheck; do
    echo "== $tool: coverage rung cases"
    timeout 150 compute-sanitizer --tool $tool --error-exitcode 9 --log-file "$OUT/${tool}_contact_rungs.log" \
        python -m pytest tests/test_contact_backward_coverage_gpu.py -q -x -k "$RUNGS" 2>&1 | tail -3
    echo "$tool rungs rc=${PIPESTATUS[0]}"; tail -3 "$OUT/${tool}_contact_rungs.log"
    echo "== $tool: fp64-oracle cases"
    timeout 120 compute-sanitizer --tool $tool --error-exitcode 9 --log-file "$OUT/${tool}_contact_oracle.log" \
        python -m pytest tests/test_contact_backward_gpu.py -q -x -k "oracle" 2>&1 | tail -3
    echo "$tool oracle rc=${PIPESTATUS[0]}"; tail -3 "$OUT/${tool}_contact_oracle.log"
done
