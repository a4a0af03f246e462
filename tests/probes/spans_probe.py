#!/usr/bin/env python3
"""Small run of the required-token routes for compute-sanitizer memcheck, checked against the span oracle: whole batch,
the chunked pipeline and device-resident input (k_mark_spans, k_candidates_spans), with spans with and without
patterns, a refused list, empty lists, and a batch re-run after a candidate pool overflow.

    tools/run_sanitizer.sh spans memcheck"""
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
from oracle import vibrato_oracle as vo  # noqa: E402
from span_oracle import SpanOracle, constraints  # noqa: E402

g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
so = SpanOracle(od, r["char.def"], r["unk.def"])
sents = ["京都東京都京都", "abcdefgh" * 20, "東京都 abc 123", "一橋大学大学院", "", "X" * 300]
SPANS = [[(0, 6, "名詞,固有名詞"), (6, 15)], [(0, 160)], [(0, 9, "NOPE"), (10, 13)], [(0, 6), (6, 21, "名詞")], [],
         [(3, 290)]]


def check(tok, ss, sps, device=False):
    e_off, e_toks = so.tokenize_batch([s.encode() for s in ss], constraints(None, sps))
    utf8, off = adv.pack(ss)
    if device:
        s_off, recs, pats = vb.Tokenizer.pack_spans(sps)
        t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64), s_off.astype(np.int64),
                                                  recs.astype(np.int64).astype(np.int32).reshape(-1)
                                                  if len(recs) else np.zeros(3, np.int32))]
        torch.cuda.synchronize()
        _, _, n = tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(ss), len(utf8),
                                            d_span_offsets=t[2].data_ptr(), d_spans=t[3].data_ptr(), n_spans=len(recs),
                                            patterns=pats)
        assert n == len(e_toks)
        return
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, spans=sps)
    assert np.array_equal(res.tok_offsets, e_off) and res.tokens.tobytes() == e_toks.astype(vb.TOKEN_DTYPE).tobytes()


for route in ("whole", "chunked", "device", "overflow"):
    tok = vb.Tokenizer.new(d)
    k = 150 if route in ("chunked", "overflow") else 1
    ss, sps = sents * k, SPANS * k
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    if route == "overflow":  # a pool sized for far fewer candidates than the batch makes: the batch runs again
        tok.set_option("pool_estimate_permille", 1)
    check(tok, ss, sps, device=route == "device")
    check(tok, ss, [[] for _ in ss], device=route == "device")
    if route != "device":
        try:
            tok.tokenize_batch(ss, spans=[[(1, 6)]] + [[] for _ in ss[1:]])  # starts inside 京
            raise SystemExit("a bad list was accepted")
        except vb.VibratoError as e:
            assert e.kind == "InvalidArgument"
        check(tok, ss, sps)
print("spans probe ok")
