#!/usr/bin/env python3
"""Small run of the sampling routes for compute-sanitizer memcheck, checked against the FFBS restatement
(tests/sampling_oracle.py) up to each sample's first ambiguous draw: whole batch, the chunked pipeline (empty
sentences at chunk edges), device-resident input and a bounded call, on the Matrix fixture and the Raw adversarial
dictionary, with ignore_space on (skipped and trailing space runs), sampling alone and next to marginals.
Kernels: k_marg_forward's sampling instantiation, k_sample_count, k_sample_write.

    tools/run_sanitizer.sh sampling memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import sampling_oracle as so  # noqa: E402
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

N, SEED = 3, 2 ** 64 - 1
g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]


def d2h(ptr, n, dtype):
    from cuda.bindings import runtime as cudart
    host = np.empty(n, dtype=dtype)
    if n:
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host


def check(bo, sents, off, recs, theta, bounds=None):
    for i, s in enumerate(sents):
        for j, (rec, _, amb) in enumerate(so.sentence_samples(bo, s.encode(), N, theta, SEED, i,
                                                             bounds[i] if bounds else ())):
            got = recs[int(off[i * N + j]):int(off[i * N + j + 1])]
            assert amb is not None or got.tobytes() == rec.tobytes(), (s, j)


def probe(d, bo, sents, theta):
    ref = None
    for route in ("whole", "chunked", "device", "marginals"):
        tok = vb.Tokenizer.new(d).ignore_space(True).sampling(N, theta, SEED)
        ss = sents
        if route == "chunked":
            tok.set_option("chunk_sentences", 64)
            ss = sents * 20 + [""] * 70 + sents * 10
        if route == "marginals":
            tok.marginals(theta)
        utf8, off = adv.pack(ss)
        if route == "device":
            t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64))]
            torch.cuda.synchronize()
            tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(ss), len(utf8))
            a, b, n = tok.last_device_samples()
            got_off, got = d2h(a, len(ss) * N + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)
        else:
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            got_off, got = res.sample_offsets.copy(), res.samples.copy()
        if route == "chunked":
            whole = vb.Tokenizer.new(d).ignore_space(True).sampling(N, theta, SEED).tokenize_batch(utf8=utf8, byte_offsets=off)
            assert got.tobytes() == whole.samples.tobytes() and np.array_equal(got_off, whole.sample_offsets)
            continue
        if ref is None:
            check(bo, ss, got_off, got, theta)
            ref = got.tobytes()
        assert got.tobytes() == ref, route


d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
sents = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "東京   都", "abc  ", "", " 東京"]
probe(d, BoundedOracle(od, r["char.def"], r["unk.def"], True), sents, 0.001)

tok = vb.Tokenizer.new(d).sampling(N, 0.001, SEED)  # bounded
bsents, bounds = ["京都東京都京都"] * 3, [[12], [], [6, 15]]
res = tok.tokenize_batch(bsents, boundaries=bounds)
check(BoundedOracle(od, r["char.def"], r["unk.def"]), bsents, res.sample_offsets, res.samples, 0.001, bounds)

w = adv.make_dictionary("wrap")
right, left, cost = w.matrix
dw = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(w.lex_csv, right, left, cost, w.char_def, w.unk_def)
ow = vo.OracleDictionary(w.lex_csv, w.matrix, w.char_def, w.unk_def)
probe(dw, BoundedOracle(ow, w.char_def, w.unk_def, True), adv.make_sentences(w, 40, seed=5, max_len=40), 1e-6)
print("sampling probe ok")
