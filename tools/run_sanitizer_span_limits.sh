#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/span_limits_probe.py, the required-token
# code at its limits (a start re-walked into the pool, far spans, 65 spans per sentence, quoted features, the
# pool-overflow re-run).
#     tools/run_sanitizer_span_limits.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 1800 compute-sanitizer --tool memcheck python tests/probes/span_limits_probe.py > "$LOG_DIR/sanitizer_memcheck_span_limits.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_span_limits.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_span_limits.log"
