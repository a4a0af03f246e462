#!/usr/bin/env python3
"""Small run of posterior decoding for compute-sanitizer memcheck, checked bit for bit against the restatement
(tests/posterior_oracle.py) fed the device's own node marginals: whole batch, the chunked pipeline (empty sentences at
chunk edges) and device-resident input, ignore_space on, with posterior text and a no-path span call.
Kernels: k_posterior_sweep and k_posterior_write, and the lw-writing instantiation of k_marg_forward.

    tools/run_sanitizer.sh posterior memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import marginal_oracle as mo  # noqa: E402
import posterior_oracle as po  # noqa: E402
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

THETA = 0.01
g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
bo = BoundedOracle(od, r["char.def"], r["unk.def"], True)
base = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "東京   都", "abc  ", "", " 東京"]


def d2h(ptr, n, dtype):
    from cuda.bindings import runtime as cudart
    host = np.empty(n, dtype=dtype)
    if n:
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host


ref = None
for route in ("whole", "chunked", "device"):
    tok = vb.Tokenizer.new(d).ignore_space(True).marginals(THETA).lattice(True).posterior(1.0)
    sents = base * 20 + [""] * 70 + base * 10
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    utf8, off = adv.pack(sents)
    if route == "device":
        t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64))]
        torch.cuda.synchronize()
        tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(sents), len(utf8))
        do, dt, dp, dg, n = tok.last_device_posterior()
        got = (d2h(do, len(sents) + 1, np.uint64), d2h(dt, n, vb.TOKEN_DTYPE), d2h(dp, n, np.float32),
               d2h(dg, len(sents), np.float64))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref))
        continue
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    got = (res.posterior_offsets, res.posterior_tokens, res.posterior_probs, res.posterior_gains)
    if ref is None:
        ref = got
        for i, s in enumerate(base):
            if not s:
                continue
            lat = mo.Lattice(bo, s.encode())
            order = [(e, k) for e in range(1, len(lat.ends)) for k in range(len(lat.ends[e]))]
            p = dict(zip(order, res.node_probs[int(res.node_offsets[i]):int(res.node_offsets[i + 1])]))
            path, v = po.sweep(lat, p, 1.0)
            a, b = int(got[0][i]), int(got[0][i + 1])
            assert got[1][a:b].tobytes() == po.records(lat, path).tobytes() and got[3][i] == v
    else:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref))

tok = vb.Tokenizer.new(d).marginals(THETA).posterior(4.0, text=True).output_mode("mecab")
res = tok.tokenize_batch(["ぬぬ京都", "", "京都東京都京都"], spans=[[(0, 6, None)], [], []])
assert res.posterior_gains[0] == -np.inf and res.posterior_gains[1] == 0.0 and res.text()[1]
print("posterior probe ok")
