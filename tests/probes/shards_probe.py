#!/usr/bin/env python3
"""Small run of the multi-device shard path for compute-sanitizer memcheck, on device 0 listed three times when the
machine has one GPU: every output on (marginals, uncertainty with boundary probabilities, the near-best lattice,
samples, posterior paths and mecab text), host and device-resident batches with required boundaries and tokens, a
sentence only the first shard holds, empty trailing shards, and device offsets past n_bytes (refused before any
shard copies its input).  Every array is checked byte for byte against the single device.
Code: multi_engine.cu (split, shard_bounds, fetch_shard, rebase_shard, the peer-copy gather) over the usual kernels.

    tools/run_sanitizer.sh shards memcheck"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from test_gpu_marginals import golden_dicts, golden_sents, shard_devices  # noqa: E402
from test_gpu_shards import bounded_batch, configured, device_call, error_of, host_call  # noqa: E402

g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
d, od, r = golden_dicts(g, True)
multi = configured(vb.Tokenizer.new(d, devices=shard_devices(3)), "all_text")
single = configured(vb.Tokenizer.new(d), "all_text")
sents, bounds, spans = bounded_batch(g, od, r)
for batch in (sents, ["京都東京都京都"], ["東京都" * 300] + golden_sents(g)):
    utf8, off = adv.pack(batch)
    assert host_call(multi, utf8, off) == host_call(single, utf8, off)
utf8, off = adv.pack(sents)
assert host_call(multi, utf8, off, boundaries=bounds, spans=spans) == host_call(single, utf8, off, boundaries=bounds,
                                                                                 spans=spans)
configured(multi, "all")
configured(single, "all")
assert device_call(multi, utf8, off, bounds=bounds, spans=spans) == device_call(single, utf8, off, bounds=bounds,
                                                                                 spans=spans)
assert error_of(lambda: device_call(multi, utf8, off, n_bytes=len(utf8) - 1)) == \
    error_of(lambda: device_call(single, utf8, off, n_bytes=len(utf8) - 1))
print("shards probe ok")
