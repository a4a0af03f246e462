#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck and racecheck over tests/probes/small_batch_probe.py,
# the k_small_batch route (one thread block: block scans and batch flags in shared memory).
#     tools/run_sanitizer_small.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
for tool in memcheck racecheck; do
    timeout 500 compute-sanitizer --tool "$tool" python tests/probes/small_batch_probe.py > "$LOG_DIR/sanitizer_${tool}_small.log" 2>&1
    echo "$tool: $LOG_DIR/sanitizer_${tool}_small.log"
    tail -4 "$LOG_DIR/sanitizer_${tool}_small.log"
done
