#!/bin/bash
# compute-sanitizer over the shipped search kernels (memcheck, racecheck, synccheck) on the small-corpus GPU tests.
# Output: ${TAG}_sanitizer_*.log in the output directory below.
TAG=${1:-r2}
mkdir -p gpurun_out
SEL='matches_oracle and (C1 or dense or manyterms or ties) or edge or prefilter or pruning or golden'
for tool in memcheck racecheck synccheck; do
  timeout 600 compute-sanitizer --tool $tool --error-exitcode 9 --print-limit 30 \
      python -m pytest tests/test_gpu_parity.py -q -m gpu -x -k "$SEL" > gpurun_out/${TAG}_sanitizer_${tool}.log 2>&1
  echo "$tool rc=$?"; tail -4 gpurun_out/${TAG}_sanitizer_${tool}.log
done
