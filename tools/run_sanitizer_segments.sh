#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/segments_probe.py, the candidate
# pool's segment encoding at its limits (move segments, 2^16-candidate sources, crowded positions, the pool-overflow
# retry the segments alone cause; k_candidates, every Viterbi kernel, k_small_batch, the marginal and lattice kernels).
#     tools/run_sanitizer_segments.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/segments_probe.py > "$LOG_DIR/sanitizer_memcheck_segments.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_segments.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_segments.log"
