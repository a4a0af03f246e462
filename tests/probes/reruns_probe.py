#!/usr/bin/env python3
"""One pass through each way the engine re-runs a batch, with every output on (tests/test_gpu_reruns.py): a pool
overflow on the whole, device-resident and chunked routes, a slot overflow, a chunk text overflow and the host result
growing; each call prints its describe()["last_reruns"] and must equal the whole-batch reference.

    tools/run_sanitizer.sh reruns memcheck"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_gpu_reruns as t  # noqa: E402

sents = t.batch(0)
for route, reason, setup, style, opts in (
        ("whole", "pool", "best", "mecab", dict(pool_estimate_permille=1)),
        ("device", "pool", "lattice", "mecab", dict(pool_estimate_permille=1)),
        ("chunked", "pool", "posterior", "mecab", dict(pool_estimate_permille=1)),
        ("chunked", "slots", "sample", "mecab", dict(chars_estimate_permille=1, pool_estimate_permille=t.BIG_PERMILLE)),
        ("chunked", "text", "lattice", t.FMT_BIG, dict(pool_estimate_permille=t.BIG_PERMILLE))):
    tok = t.make(route, setup, style, **opts)
    got, reruns = t.call(tok, route, list(sents))
    print(route, reason, setup, reruns, flush=True)
    assert reruns[reason] >= 1, reruns
    t.assert_same(got, t.reference(setup, style if route != "device" else None, sents), (route, reason))
t.test_result_grows_in_every_record_group()
print("reruns probe ok")
