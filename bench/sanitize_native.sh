#!/bin/bash
# ThreadSanitizer + AddressSanitizer/UBSan builds of the native runtime pieces that own threads (CPU only; the CUDA kernels have
# their own compute-sanitizer script, bench/sanitize.sh).  Usage: bash bench/sanitize_native.sh [outdir]
set -u
root=$(cd "$(dirname "$0")/.." && pwd)
out=${1:-$root/sanitizer_logs}
mkdir -p "$out"
tmp=$(mktemp -d)
src="$root/tests/native/data_loader_stress.cc $root/tepdist_b200/csrc/runtime/data_loader.cc"
rc=0
for san in thread "address,undefined"; do
  tag=${san%%,*}
  g++ -std=c++17 -O1 -g -fsanitize=$san -fno-omit-frame-pointer -I "$root/tepdist_b200/csrc" $src -o "$tmp/stress_$tag" -pthread || { rc=1; continue; }
  mkdir -p "$tmp/$tag"
  "$tmp/stress_$tag" "$tmp/$tag" > "$out/data_loader_$tag.log" 2>&1
  code=$?
  echo "[$tag] exit $code: $(tail -n 1 "$out/data_loader_$tag.log")"
  [ $code -ne 0 ] && rc=1
  grep -c "WARNING: ThreadSanitizer\|ERROR: AddressSanitizer\|runtime error:" "$out/data_loader_$tag.log" | sed "s/^/[$tag] sanitizer reports: /"
done
# the planner's worker pool (ILP_NUM_THREADS): ThreadSanitizer build of the planner core + a transformer-shaped graph, 1 vs 6 threads
csrc="$root/tepdist_b200/csrc"
if g++ -std=c++17 -O1 -g -fsanitize=thread -fno-omit-frame-pointer -I "$csrc" "$root/tests/native/planner_threads_stress.cc" \
     "$csrc/spmd_planner.cc" "$csrc/rules.cc" "$csrc/pbqp.cc" "$csrc/ir.cc" "$csrc/cost.cc" -o "$tmp/planner_thread" -pthread; then
  "$tmp/planner_thread" > "$out/planner_threads_thread.log" 2>&1
  code=$?
  echo "[planner] exit $code: $(tail -n 1 "$out/planner_threads_thread.log")"
  [ $code -ne 0 ] && rc=1
  grep -c "WARNING: ThreadSanitizer" "$out/planner_threads_thread.log" | sed "s/^/[planner] sanitizer reports: /"
else
  rc=1
fi
rm -rf "$tmp"
exit $rc
