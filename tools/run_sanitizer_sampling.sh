#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/sampling_probe.py, the sampling routes
# (k_marg_forward's sampling instantiation, k_sample_count, k_sample_write; whole batch, chunked, device-resident input
# and a bounded call).
#     tools/run_sanitizer_sampling.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/sampling_probe.py > "$LOG_DIR/sanitizer_memcheck_sampling.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_sampling.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_sampling.log"
