#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/uncertainty_probe.py, the
# segmentation uncertainty (k_marg_backward's uncertainty instantiation and k_boundary_probs; whole batch, chunked and
# device-resident input, levels 1 and 2).
#     tools/run_sanitizer_uncertainty.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/uncertainty_probe.py > "$LOG_DIR/sanitizer_memcheck_uncertainty.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_uncertainty.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_uncertainty.log"
