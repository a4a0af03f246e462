#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/lattice_margin_probe.py, the
# near-best lattice (k_marg_forward's R-only instantiation, k_margin_backward, k_lattice_count_margin,
# k_lattice_write_margin; whole batch, chunked and device-resident input).
#     tools/run_sanitizer_lattice_margin.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/lattice_margin_probe.py > "$LOG_DIR/sanitizer_memcheck_lattice_margin.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_lattice_margin.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_lattice_margin.log"
