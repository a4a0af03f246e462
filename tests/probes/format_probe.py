#!/usr/bin/env python3
"""Small run of the output formats (Tokenizer.output_format) for compute-sanitizer memcheck: the field-table build,
the format program staged in shared memory and interpreted by k_format_len / k_format_write (whole batch) and by
k_small_batch, with fields, quoted features, unknown words and %S; checked against tests/format_oracle.py.

    tools/run_sanitizer.sh format memcheck"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import format_oracle as fo  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
lex = r["lex.csv"] + '"ｘ,ｙ",1,1,-900,記号,"x""y",*,"p,q",,*z\n'
d = vb.SystemDictionaryBuilder.from_readers(lex, r["matrix.def"], r["char.def"], r["unk.def"])
d.reset_user_lexicon_from_reader(r["user.csv"])
od = vo.OracleDictionary(lex, r["matrix.def"], r["char.def"], r["unk.def"]).set_user_csv(r["user.csv"])
sents = [c["input"] for c in g["tokenizer_cases"]] * 4 + ["X" * 300, "", "ｘ,ｙ東京 都  ｘ,ｙ", "0123456789" * 40]
utf8, off = adv.pack(sents)
FORMATS = [("%m\\t%H\\n", None, "", "EOS\\n"),
           ("%M|%pS|%f[0,1,6]|%F\\s[1,2,30]|%c %pc %pn %pC %pL %phl %phr %s\\n", "?%m %f[3]\\n", "B%L:", "%S\\n")]
for route in ("whole", "small_batch"):
    for ign in (False, True):
        tok = vb.Tokenizer.new(d).ignore_space(ign)
        tok.set_option("chunk_sentences", 0)
        if route == "small_batch":
            tok.small_batch(64)
        tok_off, toks = od.tokenize_batch(utf8, off, ign)[:2]
        for fmt in FORMATS:
            res = tok.output_format(*fmt).tokenize_batch(utf8=utf8, byte_offsets=off)
            assert (tok.describe()["last_viterbi"] == "k_small_batch") == (route == "small_batch")
            toff, text = res.text()
            eoff, etext = fo.format_batch(od, fo.Format(*fmt), utf8, off, tok_off, toks)
            assert text == etext and (toff == eoff).all(), (route, ign, fmt)
        print(route, "ignore_space", ign, "ok", flush=True)
