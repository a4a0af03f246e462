"""Marginal probabilities on the CPU: the forward-backward restatement (tests/marginal_oracle.py) against brute-force
enumeration of every path on the golden fixture, and its properties over the adversarial dictionaries."""
import math

import pytest

import adversarial as adv
import marginal_oracle as mo
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo


def golden_oracle(golden, user=False, ignore_space=False, mgl=0):
    r = golden["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        od.set_user_csv(r["user.csv"])
    return BoundedOracle(od, r["char.def"], r["unk.def"], ignore_space, mgl)


def adversarial_oracle(family, ignore_space=False):
    if family in adv.FAMILIES:
        d, dual = adv.make_dictionary(family), False
    else:
        d, dual = adv.make_dictionary("wrap", dual=family == "dual"), family == "dual"
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=dual)
    od.set_user_csv(d.user_csv)
    return d, BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


def close(a, b, rel=1e-9, abs_=1e-12):
    return abs(a - b) <= rel * max(abs(a), abs(b)) + abs_


@pytest.mark.parametrize("case", [
    ("京都東京都京都", False, False, 0, ()),
    ("京都東京都京都", True, False, 0, ()),
    ("東京 都", False, True, 0, ()),
    ("東京   都", False, True, 0, ()),
    ("kampersanda", False, False, 9, ()),
    ("京都東京都京都", False, False, 0, (12,)),
])
@pytest.mark.parametrize("theta", [0.001, 0.01, 1.0])
def test_matches_brute_force(golden, case, theta):
    sent, user, isp, mgl, bounds = case
    bo = golden_oracle(golden, user, isp, mgl)
    lat = mo.Lattice(bo, sent.encode(), bounds)
    prob, pp, _ = mo.marginals(lat, theta)
    bprob, bpp = mo.brute_force(lat, theta)
    assert close(pp, bpp), (pp, bpp)
    for n in lat.nodes:
        assert close(prob[n], bprob[n]), (n, prob[n], bprob[n])
    if len(mo.all_paths(lat)) == 1:
        assert close(pp, 1.0) and all(close(prob[n], 1.0) for n in lat.best_path())


def test_two_paths_by_hand(golden):
    """に has two lex.csv rows and nothing else in its lattice: に,2,2,11406 and に,3,3,4481.  With matrix.def's
    connections 0->2 = 2124, 2->0 = -1959, 0->3 = 1032 and 3->0 = -2288 the two paths cost
    2124 + 11406 - 1959 = 11571 and 1032 + 4481 - 2288 = 3225, so P(the second) = 1 / (1 + exp(-theta * 8346))."""
    bo = golden_oracle(golden)
    lat = mo.Lattice(bo, "に".encode())
    paths = mo.all_paths(lat)
    assert sorted(c for c, _ in paths) == [3225, 11571]
    theta = 0.0002
    p_cheap = 1.0 / (1.0 + math.exp(-theta * (11571 - 3225)))
    prob, pp, r_eos = mo.marginals(lat, theta)
    assert r_eos == 3225 and close(pp, p_cheap)
    by_cost = {c: p[0] for c, p in paths}
    assert close(prob[by_cost[3225]], p_cheap) and close(prob[by_cost[11571]], 1.0 - p_cheap)
    assert [lat.node(n)[3] for n in lat.best_path()] == [3]  # the tokenizer's path is the cheap one
    tp, pp2 = mo.sentence_marginals(bo, "に".encode(), theta)
    assert close(tp[0], p_cheap) and close(pp2, p_cheap)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
@pytest.mark.parametrize("ignore_space", [False, True])
def test_properties(family, ignore_space):
    d, bo = adversarial_oracle(family, ignore_space)
    sents = adv.make_sentences(d, 25, seed=7, max_len=40)
    theta = 0.05 if family in adv.FAMILIES else 1e-7
    for s in sents:
        if not s:
            continue
        b = s.encode()
        lat = mo.Lattice(bo, b)
        prob, pp, _ = mo.marginals(lat, theta)
        # every character that can never be skipped is covered by exactly one node of every path
        for i, ch in enumerate(s):
            if ignore_space and ch == " ":
                continue
            cover = sum(prob[n] for n in lat.nodes if n != (0, 0) and lat.node(n)[1] <= i < n[0])
            assert abs(cover - 1.0) < 1e-9, (s, i, cover)
        for n in lat.best_path():
            # the Raw / Dual "wrap" costs make the tokenizer's i32 path costs wrap: its best path is then not a
            # minimum-cost path of the exact costs, and only prob <= 1 holds
            assert family not in adv.FAMILIES or pp <= prob[n] * (1 + 1e-9) + 1e-15
            assert prob[n] <= 1 + 1e-9


@pytest.mark.parametrize("family", ["ties", "flat_columns"])
def test_large_theta_tie_fractions(family):
    """At large theta a node's marginal is the share of minimum-cost paths through it (ties give 1/2, 1/3, ...)."""
    d, bo = adversarial_oracle(family)
    sents = [s for s in adv.make_sentences(d, 40, seed=9, max_len=30) if s]
    seen_fraction = False
    for s in sents:
        lat = mo.Lattice(bo, s.encode())
        prob, _, _ = mo.marginals(lat, 60.0)
        frac = mo.tie_fractions(lat)
        for n in lat.nodes:
            assert abs(prob[n] - float(frac[n])) < 1e-9, (s, n, prob[n], frac[n])
            seen_fraction |= 0 < frac[n] < 1
    assert seen_fraction
