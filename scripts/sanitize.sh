#!/bin/bash
# compute-sanitizer targets for the hand-written kernels (SURVEY §5.2: the reference has none).
#   scripts/sanitize.sh [memcheck|racecheck|synccheck|initcheck] [pytest -k expression]
# Run on a GPU machine (bash scripts/sanitize.sh racecheck "gemm and not large").  The wgmma / TMA paths are
# asynchronous-proxy traffic that racecheck does not model, so the interesting targets are the layer kernels
# (LRN, pooling, transform, softmax-loss, dropout, colsum, fused_update) and the epilogue's shared-memory transposes.
cd "$(dirname "$0")/.."
TOOL=${1:-memcheck}
EXPR=${2:-"lrn or pool or transform or softmax or dropout or colsum or fused_update"}
mkdir -p output
compute-sanitizer --tool "$TOOL" --error-exitcode 1 --launch-timeout 300 \
  python -m pytest tests/test_ops_gpu.py tests/test_gemm_gpu.py -q -x -p no:cacheprovider -k "$EXPR" \
  2>&1 | tail -40 | tee output/sanitize_$TOOL.log
