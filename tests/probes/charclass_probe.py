#!/usr/bin/env python3
"""Small run of the front end on the char.def fixtures of tests/charclass_fixtures.py for compute-sanitizer (memcheck
/ racecheck), checked against the oracle: k_front (shared-memory and per-warp decoding, the groupable chunk carry,
a tile too large for its text stage), k_candidates and k_candidates<BND> (boundaries inside groups), k_candidates_spans
and k_mark_spans (spans at multi-category and astral characters), k_candidate_stats (a counted run) and k_small_batch,
with the space skip on and off, and an invalid UTF-8 input.

    tools/run_sanitizer.sh charclass memcheck racecheck"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import charclass_fixtures as cf  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402
from span_oracle import Constraints, SpanOracle  # noqa: E402


def same(res, off, toks):
    assert np.array_equal(res.tok_offsets, off) and res.tokens.tobytes() == toks.tobytes()


for name in cf.FAMILIES:
    f = cf.make_family(name)
    d = vb.SystemDictionaryBuilder.from_readers(*f.sources())
    d.reset_user_lexicon_from_reader(f.user_csv)
    od = vo.OracleDictionary(*f.sources())
    od.set_user_csv(f.user_csv)
    sents = list(cf.sentences(f).values())
    utf8, off = vb.Tokenizer.pack(sents)
    for isp, mgl in ((False, 0), (True, 3)):
        e_off, e_toks, cnt = od.tokenize_batch(utf8, off, isp, mgl, want_counters=True)
        tok = vb.Tokenizer.new(d).ignore_space(isp).max_grouping_len(mgl)
        same(tok.tokenize_batch(utf8=utf8, byte_offsets=off), e_off, e_toks)
        tok.set_counting(True)
        same(tok.tokenize_batch(utf8=utf8, byte_offsets=off), e_off, e_toks)
        assert np.array_equal(tok.last_counters(), cnt)
        tok.set_counting(False)
        tile = cf.tile_batch()
        u2, o2 = vb.Tokenizer.pack(tile)
        same(tok.tokenize_batch(utf8=u2, byte_offsets=o2), *od.tokenize_batch(u2, o2, isp, mgl)[:2])
        short = [s for s in sents if len(s) <= 40]
        bounds = [[i for i in range(1, len(s.encode())) if (s.encode()[i] & 0xC0) != 0x80][::3] for s in short]
        bo = BoundedOracle(od, f.char_def, f.unk_def, isp, mgl)
        same(tok.tokenize_batch(short, boundaries=bounds), *bo.tokenize_batch([s.encode() for s in short], bounds))
        small = vb.Tokenizer.new(d).ignore_space(isp).max_grouping_len(mgl).small_batch(65536)
        u3, o3 = vb.Tokenizer.pack(short)
        same(small.tokenize_batch(utf8=u3, byte_offsets=o3), *od.tokenize_batch(u3, o3, isp, mgl)[:2])
        assert small.describe()["last_viterbi"] == "k_small_batch"
        print(name, "ignore_space", isp, flush=True)
    so = SpanOracle(od, f.char_def, f.unk_def)
    sp_sents = ["é漢ab", "\U0001F600\x00@@", "ーアー"]
    sp = [[(0, 2)], [(0, 4), (4, 5)], [(0, 6)]]
    e_off, e_toks = so.tokenize_batch([s.encode() for s in sp_sents], [Constraints((), tuple(x)) for x in sp])
    same(vb.Tokenizer.new(d).tokenize_batch(sp_sents, spans=sp), e_off, e_toks)
    print(name, "spans", flush=True)
tok = vb.Tokenizer.new(d)
try:
    tok.tokenize_batch([b"ab", "漢".encode() * 600 + b"\xe3\x81"])
    raise SystemExit("invalid UTF-8 accepted")
except vb.VibratoError as e:
    assert e.kind == "Utf8"
print("invalid UTF-8 refused", flush=True)
