"""Posterior decoding on the CPU: the restatement (tests/posterior_oracle.py) against a brute-force enumeration of every
path on the golden and adversarial lattices, with ignore_space, boundaries and required tokens: V at EOS is exactly the
largest left fold of the gains, and the chosen path attains it.  Also single-path lattices (the best path), a tie
lattice (the first entry of each row) and the empty and no-path sentences."""
import math

import numpy as np
import pytest

import adversarial as adv
import marginal_oracle as mo
import posterior_oracle as po
from span_oracle import Constraints, SpanOracle
from test_uncertainty_oracle import GOLDEN_TEXTS, adversarial_oracle, exact_oracle, golden_oracle

GAMMAS = (0.0, 0.5, 1.0, 8.0)


def check_against_brute_force(lat, theta):
    p = po.node_probs(lat, theta)
    for gamma in GAMMAS:
        path, v = po.sweep(lat, p, gamma)
        best, _, argmax = po.brute_force(lat, p, gamma)
        assert v == best, (gamma, v, best)
        assert po.fold(gamma + 1.0, p, path) == v
        assert path in argmax


def cases():
    out = [("golden", golden_oracle(), [t.encode() for t in GOLDEN_TEXTS], 0.001),
           ("golden_space", golden_oracle(ignore_space=True), [t.encode() for t in GOLDEN_TEXTS], 0.01),
           ("golden_mgl", golden_oracle(mgl=3), [t.encode() for t in GOLDEN_TEXTS], 0.001)]
    for fam in adv.FAMILIES:
        d, bo = adversarial_oracle(fam, ignore_space=fam == "ties")
        out.append((fam, bo, [s.encode() for s in adv.make_sentences(d, 14, seed=5, max_len=3 if fam == "ties" else 6)],
                    0.05))
    return out


@pytest.mark.parametrize("name,bo,texts,theta", cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_matches_brute_force(name, bo, texts, theta):
    checked = 0
    for t in texts:
        if not t:
            recs, probs, v = po.sentence_posterior(bo, t, 1.0, theta=theta)
            assert len(recs) == 0 and probs == [] and v == 0.0
            continue
        lat = mo.Lattice(bo, t)
        if not lat.ends[lat.eos_row]:
            continue
        for th in (theta, theta * 10):
            check_against_brute_force(lat, th)
        checked += 1
    assert checked >= 5


def test_bounds_and_spans():
    """Over the constrained lattice: the fold maximum, and every required boundary and span end on the path."""
    so = golden_oracle(cls=SpanOracle)
    for text, cons, ends in [
            ("京都東京都京都", Constraints((6,), ()), [2]),
            ("京都東京都京都", Constraints((), ((6, 15, None),)), [2, 5]),
            ("東京都に行った", Constraints((), ((0, 6, "名詞"),)), [2]),
            ("abcdefgh", Constraints((3, 5), ()), [3, 5])]:
        lat = mo.Lattice(so, text.encode(), cons)
        check_against_brute_force(lat, 0.001)
        for gamma in GAMMAS:
            path, _ = po.sweep(lat, po.node_probs(lat, 0.001), gamma)
            assert set(ends) <= {n[0] for n in path}, (text, gamma, path)


def test_single_path_gives_best_path():
    """One path: the posterior path is the best path, and its records are the tokenizer's."""
    zero, so = exact_oracle(adv.zero_dictionary()), golden_oracle(cls=SpanOracle)
    forced = Constraints((), ((0, 6, None), (6, 15, None), (15, 21, None)))  # a forced alignment by spans
    for bo, s, cons in ((zero, b"b", ()), (so, "京都東京都京都".encode(), forced)):
        lat = mo.Lattice(bo, s, cons)
        assert len(mo.all_paths(lat)) == 1
        for gamma in GAMMAS:
            path, v = po.sweep(lat, po.node_probs(lat, 1.0), gamma)
            assert path == lat.best_path()
            assert v == po.fold(gamma + 1.0, po.node_probs(lat, 1.0), path)


def test_tie_takes_first_entry_of_each_row():
    """Zero costs and p = 0.5 everywhere at gamma = 1: every gain is 0, so every path ties at V = 0 and the sweep takes
    entry 0 of each row back from EOS."""
    bo = exact_oracle(adv.zero_dictionary())
    for n in (1, 2, 3, 5, 8):
        lat = mo.Lattice(bo, b"a" * n)
        p = {nd: np.float32(0.5) for nd in lat.nodes}
        path, v = po.sweep(lat, p, 1.0)
        assert v == 0.0
        expect, q = [], lat.eos_row
        while q != 0:
            expect.append((q, 0))
            q = lat.node((q, 0))[0]
        assert path == expect[::-1]
        assert len(po.brute_force(lat, p, 1.0)[2]) == len(mo.all_paths(lat))


def test_underflow_takes_fewest_tokens():
    """p = 0 everywhere: every token earns -1, so the path has the fewest tokens (a a a ... -> aaa runs)."""
    bo = exact_oracle(adv.zero_dictionary())
    lat = mo.Lattice(bo, b"a" * 7)
    p = {nd: np.float32(0.0) for nd in lat.nodes}
    path, v = po.sweep(lat, p, 3.0)
    assert v == -3.0 and len(path) == 3


def test_no_path():
    """A span over hiragana, which the fixture's unk.def has no entry for, leaves no path: no tokens and -inf."""
    so = golden_oracle(cls=SpanOracle)
    recs, probs, v = po.sentence_posterior(so, "ぬぬ京都".encode(), 1.0, theta=0.01, bounds=Constraints((), ((0, 6, None),)))
    assert len(recs) == 0 and probs == [] and v == -math.inf


def test_records_of_best_path_equal_tokens():
    """Where the chosen nodes are the best path's, the records are the oracle's tokens (prefix costs included)."""
    bo = golden_oracle()
    for t in GOLDEN_TEXTS:
        lat = mo.Lattice(bo, t.encode())
        best = lat.best_path()
        rec = po.records(lat, best)
        toks = bo.tokenize(t.encode(), ())
        assert [tuple(r) for r in rec] == [tuple(x) for x in toks], t
