"""The span fixtures (tests/span_fixtures.py) on the CPU: each reaches the edge of the required-token code it is there
for, through SpanOracle's candidate trace and the segment model with span grouping (a source breaks where a record
is skipped), and the quoted-feature battery admits exactly the subsets it names.  Runs without a GPU."""
import csv

import pytest

import segment_fixtures as sf
import segment_model as sm
import span_fixtures as spf
from bounded_oracle import vo_dictionary
from span_oracle import Constraints, SpanOracle, compile_pattern, csv_fields, matches


@pytest.fixture(scope="module")
def dic():
    lex, matrix, char_def, unk_def, user, long_word = spf.make_dictionary()
    od = vo_dictionary(lex, matrix, char_def, unk_def, user)
    return od, long_word, {isp: SpanOracle(od, char_def, unk_def, isp) for isp in (False, True)}


def span_start(so, sent, spans):
    """(start slot, the encoding of its candidates with span grouping, the candidates) of the first span's word."""
    b = sent.encode()
    pos = sm.positions(so, b, Constraints((), tuple(spans)))
    a, e = len(b[:spans[0][0]].decode()), len(b[:spans[0][1]].decode())
    slot = max(s for s in pos if s <= a and all(x == e for x, _ in pos[s]))  # with ignore_space: the space's slot
    cands = pos[slot]
    enc = sm.encode(slot, cands, spans=True)
    assert decode_all(slot, enc) == cands
    if sm.n_segments(enc) <= 64:  # cand_at walks from the first segment: quadratic on the crowded starts
        assert [sm.cand_at(slot, enc, j) for j in range(len(cands))] == cands
    return slot, enc, cands


def decode_all(slot, enc):
    """Every candidate of the position, decoded segment after segment (cand_at in one pass)."""
    out, end = [], slot
    for seg in enc[0]:
        delta, c = sm.unpack_y(seg[1])
        end += delta
        out += [(end, sm.seg_record(seg, enc[1], j)) for j in range(c)]
    return out


def run_counts(slot, enc):
    return [c for _, _, c in sm.walk(slot, enc) if c]


def list_ids(od, surface, lt):
    """The word ids of the homographs of `surface` in lexicon lt, asserted contiguous (what makes sources(spans=True)
    split where span_postings does)."""
    ids = [wid for wid, end in od.common_prefix(surface, lt) if end == len(surface)]
    assert ids == list(range(ids[0], ids[0] + len(ids)))
    return ids


def test_fixture_keeps_segment_bytes():
    """Only features change (and the crowded rows are appended): ids, costs and every other byte of the segment
    fixtures' dictionary stay."""
    a = sf.make_dictionary()
    b = spf.make_dictionary()
    for x, y in zip(a, b):
        if x == y:
            continue
        xl, yl = x.splitlines(), y.splitlines()
        assert len(yl) in (len(xl), len(xl) + spf.CROWD_N)
        for p, q in zip(xl, yl):
            assert p.split(",")[:4] == q.split(",")[:4]


def test_big_lists_split_by_pattern(dic):
    od, _, sos = dic
    so = sos[False]
    seen = {}
    for s, n in spf.BIG_LISTS.items():
        lt = 1 if s == sf.BIG_USER[0] else 0
        ids = list_ids(od, s, lt)
        assert len(ids) == n
        best = sf.big_best(n)
        for name in ("all", "best", "lo", "hi"):
            pat = spf.SELECT[name]
            slot, enc, cands = span_start(so, s + "b", [(0, 1, pat)])
            keep = spf.select_expect(n, pat, best)
            if not keep:  # `hi` of the 65 535 list: the ALPHA entry instead
                assert [w for _, w in cands] == [(2 << 30) | so.unk_off[2]], (s, name)
                continue
            assert [w & 0x3FFFFFFF for _, w in cands] == [ids[0] + i for i in keep], (s, name)
            seen[(s, name)] = run_counts(slot, enc)
    assert seen[("k", "all")] == [65535] and seen[("l", "all")] == [65535, 1]
    assert seen[("m", "all")] == [65535, 2] and seen[("n", "all")] == [65535, 2]  # runs over 0xFFFF, v += c
    assert all(seen[(s, "best")] == [1] for s in spf.BIG_LISTS)
    assert all(seen[(s, "lo")] == [65535] for s in spf.BIG_LISTS)
    assert seen[("m", "hi")] == [2] and seen[("l", "hi")] == [1] and ("k", "hi") not in seen
    # the best record of the lists of 65 536 or more, and the `hi` runs, start past u16 in their list
    for s in ("l", "m", "n"):
        _, _, cands = span_start(so, s + "b", [(0, 1, spf.SELECT["best"])])
        lt = cands[0][1] >> 30
        assert (cands[0][1] & 0x3FFFFFFF) - list_ids(od, s, lt)[0] == 65535


def test_quadratic_start(dic):
    """Every second record of `m`, every third of `n`, every second BIG entry: tens of thousands of segments at one
    span start, all past kMaxSegs, so the start is walked again straight into the pool."""
    _, _, sos = dic
    so = sos[False]
    counts = {}
    for name, sent, a in spf.QUADRATIC_CASES:
        slot, enc, cands = span_start(so, sent, [(a, a + 1, spf.SELECT[name])])
        counts[(name, sent)] = (sm.n_segments(enc), len(cands))
    assert counts[("even", "mb")] == (32769, 32769)
    assert counts[("third", "nb")] == (21846, 21846)
    assert counts[("even", "Xb")] == (35000, 35000)


def test_unknown_fallback(dic):
    od, _, sos = dic
    so = sos[False]
    big = so.unk_off[4]  # BIG's first entry (DEFAULT, SPACE, ALPHA, RUN, BIG)
    assert od.feature((2 << 30) | big).startswith("BIG,0,0,1,0")
    got = {}
    for name in ("all", "none", "best", "lo", "hi", "even"):
        slot, enc, cands = span_start(so, "Xb", [(0, 1, spf.SELECT[name])])
        got[name] = run_counts(slot, enc)
        if name == "best":
            assert cands[0][1] == (2 << 30) | ((big + sf.BIG_UNK_BEST) & 0xFFFF) and big + sf.BIG_UNK_BEST > 0xFFFF
    # none matches: every entry is taken, two segments; `all` (no pattern) the same
    assert got["none"] == got["all"] == [65535, sf.BIG_UNK - 65535]
    assert got["best"] == [1] and got["lo"] == [65535] and got["hi"] == [sf.BIG_UNK - 65535]
    assert len(got["even"]) == sf.BIG_UNK // 2
    # the lexicon's `m` with a pattern that admits nothing: ALPHA's single entry
    _, _, cands = span_start(so, "mb", [(0, 1, "NOPE")])
    assert cands == [(1, (2 << 30) | so.unk_off[2])]


def test_crowded_span_starts(dic):
    """Exactly t segments at the crowded span start for t in CROWD_RUNS: kMaxSegs +- 1 and G - 1 / G / G + 1 of every
    lanes_per_sentence G; user runs before system runs."""
    od, _, sos = dic
    so = sos[False]
    ids = {lt: list_ids(od, spf.CROWD_SURFACE, lt) for lt in (0, 1)}
    assert len(ids[0]) == len(ids[1]) == spf.CROWD_N
    got = set()
    for t in spf.CROWD_RUNS:
        for sent, a in ((spf.CROWD_SURFACE + "ab", 0), ("ab" + spf.CROWD_SURFACE, 2)):
            slot, enc, cands = span_start(so, sent, [(a, a + 2, spf.crowd_pattern(t))])
            assert sm.n_segments(enc) == t, (t, sent)
            kinds = [k for k, _, _ in sm.walk(slot, enc)]
            assert kinds == sorted(kinds, key=lambda k: -k) and set(kinds) == {0, 1}
            got.add(t)
    assert {7, 8, 9} <= got and all({g - 1, g, g + 1} <= got for g in (4, 8, 16, 32))


def test_far_spans(dic):
    """The span-long unknown word ends tag.x characters on: move segments past 32 767, measured from the space run's
    slot with ignore_space; over the long user word a matching pattern keeps the word, another gives the DEFAULT
    unknown word over 4 000 characters."""
    od, long_word, sos = dic
    sents, spans, isp_sents, isp_spans = spf.far_cases(long_word)
    moves = {}
    for s, sp in zip(sents, spans):
        slot, enc, cands = span_start(sos[False], s, sp)
        a, b = sp[0][0], sp[0][1]
        assert cands and all(e == b for e, _ in cands)
        moves[(s[0], b - a)] = sm.moves(enc)
    for n in spf.FAR_LENGTHS:
        want = max(0, -(-n // sm.MAX_DELTA) - 1)
        assert moves[("Z", n)] == moves[("z", n)] == want, n
    assert moves[("Z", 32767)] == 0 and moves[("Z", 32768)] == 1 and moves[("Z", 65535)] == 2
    assert moves[("Z", 98303)] == 3
    lw = len(long_word)
    _, _, c1 = span_start(sos[False], sents[-2], spans[-2])
    _, _, c2 = span_start(sos[False], sents[-1], spans[-1])
    assert [w >> 30 for _, w in c1] == [1] and [w for _, w in c2] == [(2 << 30) | 0] and c1[0][0] == c2[0][0] == lw
    got = []
    for s, sp in zip(isp_sents, isp_spans):
        slot, enc, cands = span_start(sos[True], s, sp)
        assert slot == 0 and all(e == sp[0][1] for e, _ in cands)
        got.append((sm.moves(enc), [w >> 30 for _, w in cands]))
    assert got == [(2, [2]), (1, [1]), (1, [2])]


def test_many_spans(dic):
    """31 ... 200 spans per sentence (past one lane round of 32), spans ending at chunk edges, one span over 150 000
    characters: each span's start has its candidates, and nothing ends inside a span."""
    _, _, sos = dic
    so = sos[False]
    sents, spans = spf.many_cases()
    assert [len(sp) for sp in spans[:len(spf.MANY_COUNTS)]] == list(spf.MANY_COUNTS)
    ends = {e for a, e in spf.chunk_edge_spans()}
    assert {31, 32, 33, 63, 64, 65} <= ends
    for s, sp in zip(sents, spans):
        b = s.encode()
        lat, _, c2b = so.lattice(b, Constraints((), tuple(sp)))
        b2c = {x: i for i, x in enumerate(c2b)}
        for a, e in sp:
            assert lat[b2c[e]] and all(node[1] == b2c[a] for node in lat[b2c[e]]), (a, e)
            assert not any(lat[c] for c in range(b2c[a] + 1, b2c[e]))
    for s, sp, bnd in spf.refused_cases():
        assert len(sp) == 33
        with pytest.raises(ValueError):
            so.lattice(s.encode(), Constraints(tuple(bnd), tuple(sp)))
        so.lattice(s.encode(), Constraints((), tuple(sp[:32])))


def test_quoted_battery():
    """Each pattern admits exactly the homographs it names (or, admitting none, the unk.def entries it names)."""
    lex, matrix, char_def, unk_def = spf.make_quoted()
    od = vo_dictionary(lex, matrix, char_def, unk_def)
    so = SpanOracle(od, char_def, unk_def)
    ids = [wid for wid, end in od.common_prefix(spf.QUOTED_SURFACE) if end == 2]
    assert [od.feature(w) for w in ids] == spf.QUOTED_FEATURES
    subsets = set()
    for pat, want in spf.QUOTED_PATTERNS.items():
        c = compile_pattern(pat)
        assert [i for i, f in enumerate(spf.QUOTED_FEATURES) if matches(f, c)] == want, pat
        _, _, cands = span_start(so, "ab", [(0, 2, pat)])
        if want:
            assert [w for _, w in cands] == [ids[i] for i in want], pat
        else:
            alpha = so.unk_off[2]
            assert [w - ((2 << 30) | alpha) for _, w in cands] == spf.QUOTED_UNK_PATTERNS[pat], pat
            want = ("unk",) + tuple(spf.QUOTED_UNK_PATTERNS[pat])
        subsets.add(tuple(want))
    assert len(subsets) >= 14
    assert len(compile_pattern(",".join(["f"] * 16))) == 16 and compile_pattern(",".join(["*"] * 255 + ["w"]))[0][0] == 255


# csv_fields and Python's csv module split the same way, except where noted
CSV_DIFFERENT = {
    "": "an empty feature is one empty field; csv.reader gives no field",
}


def test_csv_fields_agree_with_csv_module():
    texts = spf.QUOTED_FEATURES + spf.QUOTED_UNK + list(spf.QUOTED_PATTERNS) + ['"a"b', '"unterminated', "a,,", ","]
    for t in texts + list(CSV_DIFFERENT):
        ours = [f.decode() for f, _ in csv_fields(t.encode())]
        theirs = next(csv.reader([t]), [])
        if t in CSV_DIFFERENT:
            assert ours != theirs
            continue
        assert ours == theirs, t
