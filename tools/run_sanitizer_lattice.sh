#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/lattice_probe.py, the lattice routes
# (k_lattice_count, k_lattice_write, the %pb format kernels; whole batch, chunked and device-resident input).
#     tools/run_sanitizer_lattice.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/lattice_probe.py > "$LOG_DIR/sanitizer_memcheck_lattice.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_lattice.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_lattice.log"
