#!/usr/bin/env python3
"""Small run of the bounded routes for compute-sanitizer memcheck, checked against the bounded oracle: whole batch,
the chunked pipeline, k_small_batch and device-resident input, with valid lists, a bad list and empty lists.
Kernels: k_mark_bounds, k_candidates<true>, k_small_batch<CONN, true>.

    tools/run_sanitizer.sh bounded memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
bo = BoundedOracle(od, r["char.def"], r["unk.def"])
sents = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "abcdefgh" * 20, "X" * 300]


def lists(ss):
    out = []
    for i, s in enumerate(ss):
        b = s.encode()
        lead = [j for j in range(1, len(b)) if (b[j] & 0xC0) != 0x80]
        out.append(lead[i % 3::3])
    return out


def check(tok, ss, bnds, device=False):
    e_off, e_toks = bo.tokenize_batch([s.encode() for s in ss], bnds)
    utf8, off = adv.pack(ss)
    if device:
        b_off, b = vb.Tokenizer.pack_bounds(bnds)
        t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64), b_off.astype(np.int64),
                                                  b.astype(np.int32) if len(b) else np.zeros(1, np.int32))]
        torch.cuda.synchronize()
        a, _, n = tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(ss), len(utf8), d_bnd_offsets=t[2].data_ptr(),
                                            d_bnd=t[3].data_ptr(), n_bnd=len(b))
        assert n == len(e_toks)
        return
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bnds)
    assert np.array_equal(res.tok_offsets, e_off) and res.tokens.tobytes() == e_toks.astype(vb.TOKEN_DTYPE).tobytes()


for route in ("whole", "chunked", "small", "device"):
    tok = vb.Tokenizer.new(d)
    ss = sents * (150 if route == "chunked" else 1)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    if route == "small":
        tok.small_batch(64)
    check(tok, ss, lists(ss), device=route == "device")
    check(tok, ss, [[] for _ in ss], device=route == "device")
    if route != "device":
        try:
            tok.tokenize_batch(ss, boundaries=[[1]] + [[] for _ in ss[1:]])  # inside 東
            raise SystemExit("a bad list was accepted")
        except vb.VibratoError as e:
            assert e.kind == "InvalidArgument"
        check(tok, ss, lists(ss))
print("bounded probe ok")
