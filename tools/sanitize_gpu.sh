#!/bin/bash
# compute-sanitizer pass over the CUDA kernels (run on a GPU box; SURVEY §5.2):
#   gpurun --timeout 1500 -- 'bash tools/sanitize_gpu.sh'
# memcheck (out-of-bounds / misaligned), racecheck (shared-memory hazards), synccheck and
# initcheck over the kernel numerics tests. Reports land in gpurun_out/sanitizer_*.log; the
# script exits non-zero if any tool reports an error.
set -u
mkdir -p gpurun_out
SAN=${COMPUTE_SANITIZER:-/usr/local/cuda/bin/compute-sanitizer}
TESTS=${SANITIZE_TESTS:-"tests/test_kernels_gpu.py tests/test_gemm_gpu.py"}
SELECT=${SANITIZE_K:-"rms_norm or layer_norm or gate_logits or adafactor or lm_head or ffn_relu or layouts"}
rc=0
for tool in ${SANITIZE_TOOLS:-memcheck racecheck synccheck initcheck}; do
  log=gpurun_out/sanitizer_${tool}.log
  timeout ${SANITIZE_TIMEOUT:-1200} "$SAN" --tool "$tool" --error-exitcode 77 --print-limit 20 \
      --launch-timeout 0 python -m pytest $TESTS -x -q -k "$SELECT" -p no:cacheprovider \
      > "$log" 2>&1
  code=$?
  errs=$(grep -c "========= .*error\|========= ERROR\|Race reported\|Invalid __" "$log" || true)
  echo "[$tool] exit=$code reports=$errs  $(grep -E 'passed|failed' "$log" | tail -1)"
  if [ "$code" -ne 0 ]; then rc=1; fi
done
exit $rc
