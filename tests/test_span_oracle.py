"""Required tokens on the CPU: the span oracle (tests/span_oracle.py) against the bounded oracle where no span is
given, against a brute-force minimum over the paths that satisfy the guarantee, and the pattern rules."""
import itertools
import json
import os

import numpy as np
import pytest

import adversarial as adv
from bounded_oracle import BoundedOracle, wrap
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, PatternError, SpanOracle, compile_pattern, matches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden_pair(user):
    with open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8") as f:
        r = json.load(f)["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        od.set_user_csv(r["user.csv"])
    return od, r["char.def"], r["unk.def"]


def adversarial_pair(family):
    d = adv.make_dictionary(family, seed=1)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od.set_user_csv(d.user_csv)
    return od, d.char_def, d.unk_def, d


def test_pattern_rules():
    assert compile_pattern(None) == [] and compile_pattern("") == [] and compile_pattern("*,*") == []
    assert compile_pattern("名詞,*,固有") == [(0, "名詞".encode()), (2, "固有".encode())]
    assert compile_pattern('"a,b",*,') == [(0, b"a,b"), (2, b"")]
    assert compile_pattern("*," * 255 + "x") == [(255, b"x")]
    with pytest.raises(PatternError) as e:
        compile_pattern("*," * 256 + "x")
    assert e.value.pos == 512
    assert len(compile_pattern(",".join("x" * 16))) == 16
    with pytest.raises(PatternError) as e:
        compile_pattern(",".join("x" * 17))
    assert e.value.pos == 32
    assert matches("名詞,一般,*", compile_pattern("名詞"))
    assert matches("名詞,一般", compile_pattern("*,一般"))
    assert not matches("名詞", compile_pattern("名詞,一般"))
    assert not matches("名詞,一般", compile_pattern("名詞,*,*,x"))
    assert matches('"a,b",c', compile_pattern('"a,b"'))


@pytest.mark.parametrize("user", [False, True])
def test_no_spans_is_the_bounded_oracle(user):
    od, cd, ud = golden_pair(user)
    so, bo = SpanOracle(od, cd, ud), BoundedOracle(od, cd, ud)
    for s, b in [("京都東京都京都", [12]), ("東京   都", [6]), ("abcdefgh", [3, 5]), ("一橋大学大学院", [])]:
        t1, t2 = so.tokenize(s.encode(), Constraints(tuple(b), ())), bo.tokenize(s.encode(), b)
        assert t1.tobytes() == t2.tobytes()


def brute_force(so, text, cons):
    """The least path cost over every segmentation of text (no ignore_space) into words whose tokens respect the
    guarantee: each span one token (from the span's own candidate rule), nothing else crossing a span or a boundary,
    and every other token a candidate the bounded lattice offers at its start."""
    n = len(text)
    sent = text.encode()
    c2b = [len(text[:i].encode()) for i in range(n + 1)]
    b2c = {b: i for i, b in enumerate(c2b)}
    spans = {b2c[a]: (b2c[e], p[0] if p else None) for a, e, *p in cons.spans}
    inside = {c for a, (e, _) in spans.items() for c in range(a + 1, e)}
    bnds = {b2c[b] for b in cons.bounds} | set(spans) | {e for e, _ in spans.values()}
    # candidates per start: those of the bounded lattice with every span end as a boundary, via its trace
    trace = []
    BoundedOracle.lattice(so, sent, sorted(c2b[c] for c in bnds if 0 < c < n), trace)
    cand = {}
    for start_node, sw, ew, widx in trace:
        cand.setdefault(sw, set()).add((ew, widx))
    for a, (e, pat) in spans.items():  # the span's own candidates, restated: rule 3
        want = [(i, f.encode()) for i, f in enumerate((pat or "").split(",")) if f != "*"] if pat else []

        def ok(widx):
            fields = so.od.feature(widx).encode().split(b",")  # no quoted fields in these dictionaries
            return all(i < len(fields) and fields[i] == f for i, f in want)

        words = [(lt << 30) | wid for lt in (1, 0) for wid, end in so.od.common_prefix(text[a:e], lt)
                 if end == e - a and ok((lt << 30) | wid)]
        if words:
            cand[a] = {(e, w) for w in words}
        else:
            c = so.od.char_info(ord(text[a]))
            ents = range(so.unk_off[(c >> 18) & 0xFF], so.unk_off[((c >> 18) & 0xFF) + 1])
            hit = [w for w in ents if ok((2 << 30) | w)]
            cand[a] = {(e, (2 << 30) | w) for w in (hit or ents)}
    best = [None]

    def walk(pos, right, cost):
        if pos == n:
            c = wrap(cost + so.conn(right, 0))
            best[0] = c if best[0] is None else min(best[0], c)
            return
        for ew, widx in sorted(cand.get(pos, ())):
            if any(pos < c < ew for c in bnds) or ew in inside:
                continue
            if pos in inside:
                continue
            left, r, wc = so.param(widx) if widx >> 30 != 2 else so.unk[[i for i in range(len(so.unk))
                                                                          if i & 0xFFFF == widx & 0xFFFF][0]]
            walk(ew, r, wrap(cost + so.conn(right, left) + wc))

    walk(0, 0, 0)
    return best[0]


def all_span_sets(n, c2b, rng, k):
    out = []
    for _ in range(k):
        pts = sorted(set(int(x) for x in rng.integers(0, n + 1, size=4)))
        sp = [(c2b[a], c2b[b]) for a, b in zip(pts, pts[1:]) if a < b and rng.random() < 0.7]
        out.append(sp)
    return out


@pytest.mark.parametrize("dictionary", ["golden", "ties", "extreme"])
def test_best_cost_is_the_brute_force_minimum(dictionary):
    if dictionary == "golden":
        od, cd, ud = golden_pair(True)
        texts = ["京都東京都京都", "abcdefgh", "東京都abc", "一橋大学大学院"]
    else:
        od, cd, ud, d = adversarial_pair(dictionary)
        texts = [s[:6] for s in adv.make_sentences(d, 6, seed=3, max_len=6) if s.strip()]
    so = SpanOracle(od, cd, ud)
    rng = np.random.default_rng(2)
    checked = 0
    for text in texts:
        n = len(text)
        c2b = [len(text[:i].encode()) for i in range(n + 1)]
        for sp in all_span_sets(n, c2b, rng, 2):
            for pat in (None, "NOPE", "名詞", "*,固有名詞", "*,普通名詞", "名詞,数"):
                cons = Constraints((), tuple((a, b, pat) for a, b in sp))
                ends, (row, _), _ = so.lattice(text.encode(), cons)
                if not ends[row]:
                    continue
                assert so.best_cost(text.encode(), cons) == brute_force(so, text, cons), (text, cons)
                checked += 1
    assert checked > 4
