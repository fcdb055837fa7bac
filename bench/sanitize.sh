#!/bin/bash
# compute-sanitizer recipe for the hand-written kernels.  STATUS: written in round 1, NOT YET EXECUTED on hardware
# (the round's GPU budget was spent before it existed) -- there are no sanitizer results anywhere in this repository.
#
# usage (one GPU, under gpurun; sanitizer slows kernels 10-100x, so only the numerics checks are run, no perf loops):
#   /usr/local/graft/bin/gpurun --timeout 1500 -- 'bash bench/sanitize.sh memcheck'
#   tools: memcheck | racecheck | synccheck | initcheck        logs: gpurun_out/sanitize_<tool>_<check>.log
#
# What each tool can and cannot tell us here:
#   memcheck  : out-of-bounds / misaligned global + shared accesses of the generic proxy (epilogues, im2col, LN, ...).
#   racecheck : SHARED-memory hazards only (P / dS tiles, LN-bwd accumulators, colsum scratch).  It does NOT see the
#               global-memory flag protocol of symm_barrier.
#   synccheck : named-barrier / __syncwarp misuse (bar.sync 1,128 in the epilogues, softmax max exchange).
#   initcheck : reads of never-written global memory (dQ accumulator).
# Unknown until run: how much of the async proxy (TMA loads, wgmma operand reads) the sanitizer models on sm_90a.
set -u
tool="${1:-memcheck}"
shift || true
checks="${*:-gemm_layouts gemm_epilogues layernorm gelu_colsum_embed xent_adam attn_fwd attn_bwd conv attn_d48}"
mkdir -p gpurun_out
rc_all=0
for c in $checks; do
  log="gpurun_out/sanitize_${tool}_${c}.log"
  timeout 600 compute-sanitizer --tool "$tool" --report-api-errors no --error-exitcode 77 --print-limit 20 \
      python tests/kernel_checks.py --one "$c" > "$log" 2>&1
  rc=$?
  echo "$tool $c rc=$rc $(grep -c 'ERROR SUMMARY\|========= Error\|Race reported\|Invalid' "$log") flagged-lines"
  [ $rc -ne 0 ] && rc_all=1
done
exit $rc_all
