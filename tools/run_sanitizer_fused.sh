#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck and racecheck over tests/probes/fused_scans_probe.py,
# the single-pass front and back kernels (tile tickets, look-back scans, staged text in shared memory).
#     tools/run_sanitizer_fused.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
for tool in memcheck racecheck; do
    timeout 500 compute-sanitizer --tool "$tool" python tests/probes/fused_scans_probe.py > "$LOG_DIR/sanitizer_${tool}_fused.log" 2>&1
    echo "$tool: $LOG_DIR/sanitizer_${tool}_fused.log"
    tail -4 "$LOG_DIR/sanitizer_${tool}_fused.log"
done
