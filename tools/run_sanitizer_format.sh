#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/format_probe.py, the output formats
# on the whole-batch route and on k_small_batch.
#     tools/run_sanitizer_format.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 500 compute-sanitizer --tool memcheck python tests/probes/format_probe.py > "$LOG_DIR/sanitizer_memcheck_format.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_format.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_format.log"
