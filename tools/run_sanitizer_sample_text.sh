#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer memcheck over tests/probes/sample_text_probe.py, the sample text
# routes (k_format_len_samples, k_format_write_samples; whole batch, chunked and the text-overflow retry).
#     tools/run_sanitizer_sample_text.sh [log directory]      (default: a new temporary directory)
cd "$(dirname "$0")/.."
LOG_DIR="${1:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
timeout 900 compute-sanitizer --tool memcheck python tests/probes/sample_text_probe.py > "$LOG_DIR/sanitizer_memcheck_sample_text.log" 2>&1
echo "memcheck: $LOG_DIR/sanitizer_memcheck_sample_text.log"
tail -4 "$LOG_DIR/sanitizer_memcheck_sample_text.log"
