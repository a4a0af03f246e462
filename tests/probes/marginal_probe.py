#!/usr/bin/env python3
"""Small run of the marginal routes for compute-sanitizer memcheck, checked against the forward-backward restatement
(tests/marginal_oracle.py): whole batch, the chunked pipeline (empty sentences at chunk edges), device-resident
input, a bounded call and a %pP output format, on the Matrix fixture and the Raw adversarial dictionary, with
ignore_space on (skipped and trailing space runs).
Kernels: k_marg_forward, k_marg_backward, k_backtrack<true>, the %pP format kernels.

    tools/run_sanitizer.sh marginal memcheck"""
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
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

THETA = 0.01
g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]


def close(got, exp):
    exp = np.asarray(exp, dtype=np.float64)
    assert got.shape == exp.shape and np.all(np.abs(got.astype(np.float64) - exp) <= 1e-3 * exp + 1e-6)


def probe(d, bo, sents, theta):
    e_tp, e_pp = mo.batch_marginals(bo, [s.encode() for s in sents], theta)
    for route in ("whole", "chunked", "device"):
        tok = vb.Tokenizer.new(d).ignore_space(True).marginals(theta)
        ss = sents
        if route == "chunked":
            tok.set_option("chunk_sentences", 64)
            ss = sents * 20 + [""] * 70 + sents * 10
        utf8, off = adv.pack(ss)
        if route == "device":
            t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64))]
            torch.cuda.synchronize()
            _, _, n = tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(ss), len(utf8))
            tp, pp = tok.last_device_marginals()
            host = np.empty(n, np.float32)
            if n:
                from cuda.bindings import runtime as cudart
                (err,) = cudart.cudaMemcpy(host.ctypes.data, tp, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
                assert int(err) == 0
            close(host, e_tp)
            continue
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        if route == "whole":
            close(res.token_probs, e_tp)
            close(res.path_probs, e_pp)
        else:
            ref = vb.Tokenizer.new(d).ignore_space(True).marginals(theta).tokenize_batch(utf8=utf8, byte_offsets=off,
                                                                                          boundaries=[[] for _ in ss])
            assert res.token_probs.tobytes() == ref.token_probs.tobytes()


d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
sents = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "東京   都", "abc  ", "", " 東京"]
probe(d, BoundedOracle(od, r["char.def"], r["unk.def"], True), sents, THETA)

tok = vb.Tokenizer.new(d).marginals(THETA)  # bounded, and a %pP format
res = tok.tokenize_batch(["京都東京都京都"] * 3, boundaries=[[12], [], [6, 15]])
assert res.token_probs is not None and np.all(np.isfinite(res.token_probs))
_, text = tok.output_format("%m\t%pP\n").tokenize_batch(sents).text()
assert text.count(b"\n") > len(sents)

w = adv.make_dictionary("wrap")
right, left, cost = w.matrix
dw = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(w.lex_csv, right, left, cost, w.char_def, w.unk_def)
ow = vo.OracleDictionary(w.lex_csv, w.matrix, w.char_def, w.unk_def)
probe(dw, BoundedOracle(ow, w.char_def, w.unk_def, True), adv.make_sentences(w, 40, seed=5, max_len=40), 1e-6)
print("marginal probe ok")
