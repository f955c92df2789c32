#!/bin/bash
# Runs every -m gpu test file in its own process (a trapped kernel poisons only its own CUDA context),
# each under a hard timeout so a protocol bug can never hang the GPU.
cd "$(dirname "$0")/.."
rc=0
for f in tests/test_*_gpu.py tests/test_band_surface.py; do
  echo "=== $f"
  timeout 600 python -m pytest "$f" -q -m gpu -x --tb=short -s 2>&1 | tail -40
  r=${PIPESTATUS[0]}
  [ "$r" -ne 0 ] && rc=$r
done
exit $rc
