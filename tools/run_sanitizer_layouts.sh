#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck and racecheck over tests/probes/layouts_probe.py,
# marginals, lattice and sampling on the layout lanes_per_sentence 4 / sort_by_length 2 (k_viterbi2<4>,
# k_marg_forward / k_marg_backward through Batch::order, k_lattice_*, k_sample_*; whole batch and device-resident).
#     tools/run_sanitizer_layouts.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
for tool in memcheck racecheck; do
    timeout 900 compute-sanitizer --tool "$tool" python tests/probes/layouts_probe.py > "$LOG_DIR/sanitizer_${tool}_layouts.log" 2>&1
    echo "$tool: $LOG_DIR/sanitizer_${tool}_layouts.log"
    tail -4 "$LOG_DIR/sanitizer_${tool}_layouts.log"
done
