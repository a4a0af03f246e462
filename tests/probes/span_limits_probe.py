#!/usr/bin/env python3
"""Small run of the required-token code at its limits for compute-sanitizer memcheck, checked against the span oracle:
a start with more segments than the shared-memory pass keeps (re-walked into the pool), far spans with move segments,
65 spans in one sentence, the quoted-feature battery, and the pool-overflow re-run.

    tools/run_sanitizer.sh span_limits memcheck"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import segment_fixtures as sf  # noqa: E402
import span_fixtures as spf  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402
from span_oracle import Constraints, SpanOracle  # noqa: E402


def check(tok, so, sents, spans):
    e_off, e_toks = so.tokenize_batch([s.encode() for s in sents], [Constraints((), tuple(sp)) for sp in spans])
    res = tok.tokenize_batch(sents, spans=spans)
    assert (res.tok_offsets == e_off).all() and res.tokens.tobytes() == e_toks.astype(vb.TOKEN_DTYPE).tobytes()


lex, matrix, char_def, unk_def, user, long_word = spf.make_dictionary()
d = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
so = SpanOracle(vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user), char_def, unk_def)
crowd, crowd_spans = spf.crowd_cases()
rewalk = (crowd[-7:], crowd_spans[-7:])  # 31 / 32 / 33 segments at one start, past kMaxSegs, and three crowded spans
big, big_spans = spf.big_spans([("all", "mb", 0), ("hi", "mb", 0), ("none", "Xb", 0), ("best", "lb", 0)])
far = (["Z" * 32768 + "Zab", "z" * 65575], [[(0, 32768)], [(20, 65555)]])
many_s, many_sp = spf.many_cases()
many = ([many_s[4]], [many_sp[4][:65]])
for what, (sents, spans) in (("rewalk", rewalk), ("big", (big, big_spans)), ("far", far), ("many", many)):
    for route in ("whole", "overflow"):
        tok = vb.Tokenizer.new(d).lattice(True)
        if route == "overflow":  # the smallest pool, and 70 000 BIG candidates in front that outgrow it
            tok.set_option("pool_estimate_permille", 1)
            sents, spans = ["Xb"] + sents, [[(0, 1)]] + spans
        check(tok, so, sents, spans)
    print(what, "ok", flush=True)
tok = vb.Tokenizer.new(d)
try:
    s, sp, bnd = spf.refused_cases()[0]
    tok.tokenize_batch([s], spans=[sp], boundaries=[bnd])
    raise SystemExit("a bad list was accepted")
except vb.VibratoError as e:
    assert e.kind == "InvalidArgument"
check(tok, so, *rewalk)
qlex, qmatrix, qchar, qunk = spf.make_quoted()
qd = vb.SystemDictionaryBuilder.from_readers(qlex, qmatrix, qchar, qunk)
qso = SpanOracle(vo.OracleDictionary(qlex, qmatrix, qchar, qunk), qchar, qunk)
check(vb.Tokenizer.new(qd).lattice(True), qso, *spf.quoted_cases())
print("span limits probe ok")
