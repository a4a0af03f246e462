#!/usr/bin/env python3
"""Small run of the single-pass front and back kernels (k_front, k_backtrack) for compute-sanitizer (memcheck /
racecheck), checked against the oracle: the inputs of tests/test_gpu_fused_scans.py on the whole-batch, chunked and
compact routes, an input error in the last tile and the slot-overflow re-run.
Kernels: k_front and k_backtrack (tile tickets, look-back scans, staged text in shared memory).

    tools/run_sanitizer.sh fused_scans memcheck racecheck"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import vibrato_b200 as vb  # noqa: E402
from test_gpu_fused_scans import base_sents, check, make, run  # noqa: E402
from test_gpu_parity import dicts  # noqa: E402

with open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8") as f:
    golden = json.load(f)
pool = base_sents(golden)
long = [pool[i % len(pool)] for i in range(100)]
long[40] = "東京都に" * 1500
long[70] = "X" * 300 + "9" * 300
for route in ("whole", "chunked", "compact"):
    d, od = dicts(golden, True)
    for n in (0, 1, 33, 257):
        check(d, od, [pool[(i * 7) % len(pool)] for i in range(n)], route)
    check(d, od, long, route)
    tok = make(d, route)
    tok.set_option("chars_estimate_permille", 1)
    check(d, od, ["X" * 50, "9" * 30, "東京都"] * 100, route, tok)
d, _ = dicts(golden)
utf8, off = vb.Tokenizer.pack(long)
bad = utf8.copy()
bad[int(off[-2])] = 0xFF
try:
    run(make(d, "whole"), "whole", bad, off)
    accepted = True
except Exception:
    accepted = False
assert not accepted, "invalid UTF-8 in the last tile was accepted"
print("fused scans probe ok")
