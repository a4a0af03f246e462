#!/usr/bin/env python3
"""Small run of the k_small_batch route for compute-sanitizer (memcheck / racecheck), checked against the oracle:
the block scans, the shared batch flags and the per-warp stages of the one-block kernel, on the Matrix, Raw and Dual
connectors, with the output stage, compact records, an input error and the overflow fallback.

    tools/run_sanitizer.sh small_batch memcheck racecheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402


def run(tok, od, sents, ignore_space=False, mode=None):
    utf8, off = adv.pack(sents)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert tok.describe()["last_viterbi"] == "k_small_batch" and tok.last_launch_count() == 1
    tok_off, toks = od.tokenize_batch(utf8, off, ignore_space)[:2]
    assert np.array_equal(res.tok_offsets, tok_off) and res.tokens.tobytes() == toks.tobytes()
    if mode:
        assert res.text()[1] == vo.format_batch(od, utf8, off, tok_off, toks, mode)[1]
    return res


g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
d.reset_user_lexicon_from_reader(r["user.csv"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"]).set_user_csv(r["user.csv"])
sents = [c["input"] for c in g["tokenizer_cases"]] * 4 + ["X" * 300, "", "0123456789" * 40, "東京 都  "]
for ign in (False, True):
    tok = vb.Tokenizer.new(d).ignore_space(ign).max_grouping_len(24 if ign else 0).small_batch(64)
    run(tok, od, sents, ign)
    run(tok, od, sents[:1], ign)
    run(tok, od, [], ign)
    for mode in ("mecab", "wakati", "detail"):
        tok.output_mode(mode)
        run(tok, od, sents, ign, mode)
    tok.output_mode(None)
    print("fixture ignore_space", ign, flush=True)
tok = vb.Tokenizer.new(d).small_batch(64).compact_tokens(True)
res = tok.tokenize_batch(sents)
assert tok.describe()["last_viterbi"] == "k_small_batch"
print("compact", res.n_tokens, flush=True)
try:
    tok.tokenize_batch(utf8=np.frombuffer(b"ab\xffcd", dtype=np.uint8), byte_offsets=np.array([0, 2, 5], dtype=np.uint64))
    raise SystemExit("invalid UTF-8 accepted")
except vb.VibratoError:
    pass
print("invalid UTF-8 refused", flush=True)
for connector in ("matrix", "raw", "dual"):
    a = adv.make_dictionary("ties" if connector == "matrix" else "wrap", dual=connector == "dual")
    if connector == "matrix":
        dev = vb.SystemDictionaryBuilder.from_readers(a.lex_csv, a.matrix, a.char_def, a.unk_def)
    else:
        dev = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(a.lex_csv, *a.matrix, a.char_def, a.unk_def,
                                                                       dual_connector=connector == "dual")
    oa = vo.OracleDictionary(a.lex_csv, a.matrix, a.char_def, a.unk_def, dual_connector=connector == "dual")
    dev.reset_user_lexicon_from_reader(a.user_csv)
    oa.set_user_csv(a.user_csv)
    tok = vb.Tokenizer.new(dev).ignore_space(True).small_batch(64)
    run(tok, oa, adv.make_sentences(a, 64, seed=3, max_len=60), True)
    print("adversarial", connector, flush=True)
# the candidate pool overflows: the kernel stops, the batch runs again on the usual route
lex = "".join(f"a,0,0,{i % 7},A{i}\n" for i in range(200))
src = (lex, "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n")
tok = vb.Tokenizer.new(vb.SystemDictionaryBuilder.from_readers(*src)).small_batch(64)
u8, o = adv.pack(["a" * 1000])
res = tok.tokenize_batch(utf8=u8, byte_offsets=o)
assert tok.describe()["last_viterbi"] == "k_viterbi2"
assert res.tokens.tobytes() == vo.OracleDictionary(*src).tokenize_batch(u8, o)[1].tobytes()
print("overflow fallback ok", flush=True)
