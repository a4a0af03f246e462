"""Segmentation uncertainty on the CPU: the restatement (tests/uncertainty_oracle.py) against a brute-force enumeration
of every path (entropy, best-path log-probability, boundary sums, expected token count) on the golden and adversarial
lattices, with boundaries and required tokens, and against exact values: unit-cost lattices at theta = ln 2 / unit,
zero-cost lattices (H = ln #paths) and single paths (H = 0)."""
import json
import math
import os

import pytest

import adversarial as adv
import marginal_oracle as mo
import uncertainty_oracle as uo
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_TEXTS = ["京都東京都京都", "東京都に行った", "abcdefgh", "東京   都", "一橋大学大学院", "に", "kampersanda"]


def golden_oracle(user=True, ignore_space=False, mgl=0, cls=BoundedOracle):
    with open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8") as f:
        r = json.load(f)["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        od.set_user_csv(r["user.csv"])
    return cls(od, r["char.def"], r["unk.def"], ignore_space, mgl)


def adversarial_oracle(family, ignore_space=False):
    d = adv.make_dictionary(family)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od.set_user_csv(d.user_csv)
    return d, BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


def close(a, b, rel=1e-9, abs_=1e-9):
    return abs(a - b) <= rel * max(abs(a), abs(b)) + abs_


def check_against_brute_force(lat, theta):
    h, lpp, bnd = uo.uncertainty(lat, theta)
    bh, blpp, bbnd, tokens = uo.brute_force(lat, theta)
    assert close(h, bh), (h, bh)
    assert close(lpp, blpp), (lpp, blpp)
    assert len(bnd) == len(bbnd) == len(lat.ends)
    assert all(close(x, y) for x, y in zip(bnd, bbnd)), (bnd, bbnd)
    assert close(sum(bnd[1:]), tokens)
    assert h >= -1e-12 and lpp <= 1e-12
    _, pp, _ = mo.marginals(lat, theta)
    assert close(math.exp(lpp), pp, abs_=1e-300)
    return h


def cases():
    out = [("golden", golden_oracle(), [t.encode() for t in GOLDEN_TEXTS], 0.001)]
    out.append(("golden_space", golden_oracle(ignore_space=True), [t.encode() for t in GOLDEN_TEXTS], 0.01))
    out.append(("golden_mgl", golden_oracle(mgl=3), [t.encode() for t in GOLDEN_TEXTS], 0.001))
    for fam in adv.FAMILIES:  # "ties" has tens of homographs per row: its short sentences have 10^5 paths
        d, bo = adversarial_oracle(fam, ignore_space=fam == "ties")
        out.append((fam, bo, [s.encode() for s in adv.make_sentences(d, 14, seed=5, max_len=3 if fam == "ties" else 6)],
                    0.05))
    return out


@pytest.mark.parametrize("name,bo,texts,theta", cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_matches_brute_force(name, bo, texts, theta):
    checked = 0
    for t in texts:
        if not t:
            assert uo.sentence_uncertainty(bo, t, theta) == (0.0, 0.0, [1.0])
            continue
        lat = mo.Lattice(bo, t)
        for th in (theta, theta * 10):
            check_against_brute_force(lat, th)
        checked += 1
    assert checked >= 5


def test_bounds_and_spans():
    """Over the constrained lattice: brute force, required boundaries and span ends at 1, span interiors at 0."""
    so = golden_oracle(cls=SpanOracle)
    for text, cons, ends, inside in [
            ("京都東京都京都", Constraints((6,), ()), [2], []),
            ("京都東京都京都", Constraints((), ((6, 15, None),)), [2, 5], [3, 4]),
            ("東京都に行った", Constraints((), ((0, 6, "名詞"),)), [2], [1]),
            ("abcdefgh", Constraints((3, 5), ()), [3, 5], [])]:
        lat = mo.Lattice(so, text.encode(), cons)
        check_against_brute_force(lat, 0.001)
        _, _, bnd = uo.uncertainty(lat, 0.001)
        assert all(close(bnd[p], 1.0, abs_=1e-12) for p in ends), (text, bnd)
        assert all(bnd[p] == 0.0 for p in inside), (text, bnd)
        assert close(bnd[-1], 1.0, abs_=1e-12) and bnd[0] == 1.0


def test_no_path():
    """A span over hiragana, which the fixture's unk.def has no entry for, leaves no path: 0, -inf and all-zero
    boundaries."""
    so = golden_oracle(cls=SpanOracle)
    lat = mo.Lattice(so, "ぬぬ京都".encode(), Constraints((), ((0, 6, None),)))
    assert not uo.has_path(lat) and not mo.all_paths(lat)
    h, lpp, bnd = uo.uncertainty(lat, 0.01)
    assert h == 0.0 and lpp == -math.inf and bnd == [0.0] * 5
    assert uo.brute_force(lat, 0.01)[:3] == (h, lpp, bnd)


def exact_oracle(d, ignore_space=False):
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    if d.user_csv:
        od.set_user_csv(d.user_csv)
    return BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


@pytest.mark.parametrize("n", [1, 2, 3, 10, 40, 200])
def test_zero_costs_give_log_path_count(n):
    """Zero-cost dictionary: T(n) (tribonacci) equally likely paths, so H = ln T(n) and ln P(best) = -ln T(n), at any
    theta; the float64 restatement within 1e-12 relative."""
    bo = exact_oracle(adv.zero_dictionary())
    lat = mo.Lattice(bo, b"a" * n)
    a, b, c = 0, 0, 1
    for _ in range(n):
        a, b, c = b, c, a + b + c
    ln_t = math.log(c)
    h, lpp = uo.exact_uncertainty(lat, 1)
    assert close(h, ln_t, rel=1e-15, abs_=0) and close(lpp, -ln_t, rel=1e-15, abs_=0)
    for theta in (1e-6, 0.01, 50.0):
        h2, lpp2, bnd = uo.uncertainty(lat, theta)
        assert close(h2, h, rel=1e-12, abs_=1e-12) and close(lpp2, lpp, rel=1e-12, abs_=1e-12)
        assert bnd[0] == 1.0 and close(bnd[-1], 1.0, abs_=1e-12)


def test_single_path_has_no_entropy():
    """One path: H = 0 and ln P(best) = 0 exactly in the exact restatement, and to rounding in float64."""
    bo = exact_oracle(adv.zero_dictionary())
    lat = mo.Lattice(bo, b"b")
    assert len(mo.all_paths(lat)) == 1
    assert uo.exact_uncertainty(lat, 1) == (0.0, 0.0)
    h, lpp, bnd = uo.uncertainty(lat, 1.0)
    assert h == 0.0 and lpp == 0.0 and bnd == [1.0, 1.0]


@pytest.mark.parametrize("ignore_space", [False, True])
def test_exact_pow2(ignore_space):
    """Costs that are multiples of 64 across i16 at theta = ln 2 / 64: exact rationals against the float64
    restatement (1e-10 relative) and the brute force where it is affordable."""
    d = adv.make_dictionary("pow2")
    bo = exact_oracle(d, ignore_space)
    theta = math.log(2) / adv.POW2_UNIT
    checked = 0
    for s in adv.make_sentences(d, 30, seed=3, max_len=10):
        if not s.strip(" ") and ignore_space or not s:
            continue
        lat = mo.Lattice(bo, s.encode())
        h, lpp = uo.exact_uncertainty(lat, adv.POW2_UNIT)
        h2, lpp2, _ = uo.uncertainty(lat, theta)
        assert close(h2, h, rel=1e-10, abs_=1e-10) and close(lpp2, lpp, rel=1e-10, abs_=1e-10), (s, h, h2, lpp, lpp2)
        if len(s) <= 4:
            bh, blpp, _, _ = uo.brute_force(lat, theta)
            assert close(bh, h) and close(blpp, lpp)
        checked += 1
    assert checked > 15
