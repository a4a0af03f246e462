#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/bounded_probe.py, the bounded routes
# (k_mark_bounds, k_candidates<true>, k_small_batch<CONN, true>, device-resident boundary lists).
#     tools/run_sanitizer_bounded.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/bounded_probe.py > "$LOG_DIR/sanitizer_memcheck_bounded.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_bounded.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_bounded.log"
