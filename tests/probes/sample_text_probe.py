#!/usr/bin/env python3
"""Small run of sample text ("sample_text" = 1) for compute-sanitizer memcheck: the whole batch, the chunked
pipeline (empty sentences at chunk edges) and the text-overflow retry, with a format that prints the "prev"
directives and BOS / EOS with %S %L, and -O mecab / wakati.  Each route's text is checked against the whole batch.
Kernels: k_format_len_samples, k_format_write_samples.

    tools/run_sanitizer.sh sample_text memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import vibrato_b200 as vb  # noqa: E402

N, SEED, THETA = 3, 2 ** 64 - 1, 0.01
FMT = ("[%M|%pS|%pn|%pC|%pL]", None, "<%S %L>", "\n")
g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]


def text(tok, sents):
    res = tok.tokenize_batch(sents)
    out = res.text()
    res.close()
    return out


def style(tok, s):
    return tok.output_mode(s) if isinstance(s, str) else tok.output_format(*s)


d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
d.reset_user_lexicon_from_reader(r["user.csv"])
sents = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "東京   都", "abc  ", "", " 東京"]
for s in ("mecab", "wakati", FMT):
    whole_sents = sents * 20 + [""] * 70 + sents * 10
    ref = text(style(vb.Tokenizer.new(d).ignore_space(True).sampling(N, THETA, SEED, text=True), s), whole_sents)
    tok = style(vb.Tokenizer.new(d).ignore_space(True).sampling(N, THETA, SEED, text=True), s)
    tok.set_option("chunk_sentences", 64)
    got = text(tok, whole_sents)
    assert got[1] == ref[1] and np.array_equal(got[0], ref[0]), s

# the retry: one-character surfaces with 1-2 KB features outgrow a fresh tokenizer's chunk text buffers
rng = np.random.default_rng(8)
chars = "abcdefghijklmnop"
lex = "".join(f"{c},0,0,{10 * i},{c}:" + "x" * int(rng.integers(1000, 2000)) + "\n" for i, c in enumerate(chars))
dl = vb.SystemDictionaryBuilder.from_readers(lex, "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n")
lsents = ["".join(rng.choice(list(chars), size=int(rng.integers(0, 30)))) for _ in range(600)]
ref = text(vb.Tokenizer.new(dl).sampling(N, THETA, SEED, text=True).output_format(*FMT), lsents)
tok = vb.Tokenizer.new(dl).sampling(N, THETA, SEED, text=True).output_format(*FMT)
tok.set_option("chunk_sentences", 128)
got = text(tok, lsents)
assert got[1] == ref[1] and np.array_equal(got[0], ref[0])
print("sample text probe ok")
