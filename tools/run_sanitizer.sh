#!/bin/bash
# Developer tool (needs a CUDA GPU): compute-sanitizer over one probe, tests/probes/<probe>_probe.py (its docstring
# says what it covers), once per tool; prints where each log went and its last four lines.
#     tools/run_sanitizer.sh [-o log directory] probe tool [tool ...]      (default: a new temporary directory)
#     tools/run_sanitizer.sh lattice_margin memcheck
#     tools/run_sanitizer.sh -o logs small_batch memcheck racecheck
cd "$(dirname "$0")/.."
LOG_DIR=
if [ "$1" = -o ]; then
    LOG_DIR="$2"
    shift 2
fi
probe="$1"
shift
if [ ! -f "tests/probes/${probe}_probe.py" ] || [ $# -eq 0 ]; then
    echo "usage: $0 [-o log directory] probe tool [tool ...]   (probe: tests/probes/<probe>_probe.py)" >&2
    exit 2
fi
LOG_DIR="${LOG_DIR:-$(mktemp -d)}"
mkdir -p "$LOG_DIR"
for tool in "$@"; do
    log="$LOG_DIR/sanitizer_${tool}_${probe}.log"
    # long enough for the slowest probe, span_limits under memcheck
    timeout 1800 compute-sanitizer --tool "$tool" python "tests/probes/${probe}_probe.py" > "$log" 2>&1
    echo "$tool: $log"
    tail -4 "$log"
done
