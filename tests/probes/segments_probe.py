#!/usr/bin/env python3
"""Small run of the segment-encoded candidate pool at its limits for compute-sanitizer memcheck, checked against the
oracle: far end slots (move segments), 2^16-candidate sources, crowded positions (tests/segment_fixtures.py), on
the whole batch, k_small_batch and with marginals and the lattice on, then the pool-overflow retry that only the
segments cause.
Kernels: k_candidates, every Viterbi kernel, k_small_batch, the marginal and lattice kernels.

    tools/run_sanitizer.sh segments memcheck"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import segment_fixtures as sf  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

lex, matrix, char_def, unk_def, user, _ = sf.make_dictionary()
d = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)


def check(tok, sents):
    utf8, off = adv.pack(sents)
    e_off, e_toks, _ = od.tokenize_batch(utf8, off)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert np.array_equal(res.tok_offsets, e_off)
    for name in vb.TOKEN_DTYPE.names:
        assert np.array_equal(res.tokens[name], e_toks[name]), name
    return tok.describe()["last_viterbi"]


far = ["Z" * 70000, "z" * 40000, sf.SPACE_RUN + "ab z"]
packed = sf.crowd_sentences() + sf.big_sentences()
for kernel in (0, 1):
    tok = vb.Tokenizer.new(d)
    tok.set_option("viterbi_kernel", kernel)
    check(tok, far)
    check(tok, packed)
small = vb.Tokenizer.new(d)
small.small_batch(64)
assert check(small, sf.crowd_sentences()) == "k_small_batch"
assert check(small, ["bmbXb"]) != "k_small_batch"
marg = vb.Tokenizer.new(d).marginals(0.01)
marg.lattice(True)
check(marg, far[:1] + packed)
retry = vb.Tokenizer.new(d)
retry.set_option("pool_estimate_permille", sf.OUTNUMBER_PERMILLE)
check(retry, sf.OUTNUMBER_SENTENCES)
print("segments probe ok")
