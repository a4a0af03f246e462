#!/usr/bin/env python3
"""Small run of the segmentation uncertainty for compute-sanitizer memcheck, checked against the restatement
(tests/uncertainty_oracle.py): whole batch, the chunked pipeline (empty sentences at chunk edges) and device-resident
input, at levels 1 and 2, ignore_space on, with a no-path span call.
Kernels: k_marg_backward's uncertainty instantiation and k_boundary_probs.

    tools/run_sanitizer.sh uncertainty memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import marginal_oracle as mo  # noqa: E402
import torch  # noqa: E402
import uncertainty_oracle as uo  # noqa: E402
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


def close(a, b):
    return np.allclose(a, b, rtol=1e-9, atol=1e-9)


for level in (1, 2):
    for route in ("whole", "chunked", "device"):
        tok = vb.Tokenizer.new(d).ignore_space(True).marginals(THETA).uncertainty(True, boundary_probs=level == 2)
        sents = base
        if route == "chunked":
            tok.set_option("chunk_sentences", 64)
            sents = base * 20 + [""] * 70 + base * 10
        e_ent, e_lpp, e_off, e_bnd = uo.batch_uncertainty(bo, [s.encode() for s in sents], THETA)
        utf8, off = adv.pack(sents)
        if route == "device":
            t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64))]
            torch.cuda.synchronize()
            tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(sents), len(utf8))
            de, dl, dbo, dbp, npos = tok.last_device_uncertainty()
            got = (d2h(de, len(sents), np.float64), d2h(dl, len(sents), np.float64),
                   d2h(dbo, len(sents) + 1, np.uint64) if dbo else None, d2h(dbp, npos, np.float32) if dbp else None)
        else:
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            got = (res.entropies, res.log_path_probs, res.boundary_offsets, res.boundary_probs)
        assert close(got[0], e_ent) and close(got[1], e_lpp)
        if level == 2:
            assert np.array_equal(got[2], e_off)
            mo.assert_f32_close(got[3], e_bnd)
        else:
            assert got[2] is None and got[3] is None

tok = vb.Tokenizer.new(d).marginals(THETA).uncertainty(True, boundary_probs=True)
res = tok.tokenize_batch(["ぬぬ京都", ""], spans=[[(0, 6, None)], []])
assert res.log_path_probs[0] == -np.inf and res.boundary_probs.tolist() == [0.0] * 5 + [1.0]
print("uncertainty probe ok")
