#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/spans_probe.py, the required-token
# routes (k_mark_spans, k_candidates_spans; whole batch, chunked, device-resident span lists, pool-overflow re-run).
#     tools/run_sanitizer_spans.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/spans_probe.py > "$LOG_DIR/sanitizer_memcheck_spans.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_spans.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_spans.log"
