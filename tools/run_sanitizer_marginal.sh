#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/marginal_probe.py, the marginal
# routes (k_marg_forward, k_marg_backward, k_backtrack<true>, the %pP format kernels; whole batch, chunked,
# device-resident and bounded input).
#     tools/run_sanitizer_marginal.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/marginal_probe.py > "$LOG_DIR/sanitizer_memcheck_marginal.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_marginal.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_marginal.log"
