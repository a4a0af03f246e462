"""Marginal probabilities on the CPU: the forward-backward restatement (tests/marginal_oracle.py) against brute-force
enumeration of every path on the golden fixture, its properties over the adversarial dictionaries, and its float32
rounding against the exact marginals of the zero-cost and power-of-two dictionaries."""
import math

import numpy as np
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


def exact_oracle(d, ignore_space=False):
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    if d.user_csv:
        od.set_user_csv(d.user_csv)
    return BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


def tribonacci(n):
    a, b, c = 0, 0, 1  # T(0) = 1: the empty path
    for _ in range(n):
        a, b, c = b, c, a + b + c
    return c


def check_f64_against_exact(lat, theta, exact):
    prob, pp, _ = mo.marginals(lat, theta)
    e_prob, e_pp = exact
    got = np.array([prob[n] for n in lat.nodes] + [pp], dtype=np.float32)
    mo.assert_f32_close(got, [e_prob[n] for n in lat.nodes] + [e_pp], ulps=1)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 33, 160, 1000, 1200, 20000])
def test_exact_path_counts(n):
    """On the zero-cost dictionary a sentence of n `a` has T(n) (tribonacci) paths, path_prob = 1 / T(n), and
    marginals() (float64) rounds to the exact float32 at any theta: through float32's subnormals (n = 160) and past
    10^308 paths (n = 1200: 1.7e317; n = 20 000: about 10^5292), where only the log-domain sums stay finite."""
    bo = exact_oracle(adv.zero_dictionary())
    lat = mo.Lattice(bo, b"a" * n)
    exact = mo.exact_marginals(lat, 1)
    assert exact[1] == 1 / tribonacci(n)
    if n >= 1200:
        assert tribonacci(n) > 10 ** 308
    for theta in (1e-6, 0.01, 50.0):
        check_f64_against_exact(lat, theta, exact)
    if n == 160:
        assert 0 < np.float32(exact[1]) < np.finfo(np.float32).tiny  # a float32 subnormal


@pytest.mark.parametrize("ignore_space", [False, True])
def test_exact_zero_mixed(ignore_space):
    """Zero-cost sentences with unknown words (`b` groups, other characters) and space runs: marginals() within one
    float32 step of the exact value, and the large-theta tie fractions equal to it (every path is a minimum)."""
    d = adv.zero_dictionary()
    bo = exact_oracle(d, ignore_space)
    sents = adv.make_sentences(d, 80, seed=4, max_len=300) + ["ab" * 50, "b" * 40, "aab  a", "  "]
    for s in sents:
        if not s.strip(" ") and ignore_space or not s:
            continue
        lat = mo.Lattice(bo, s.encode())
        exact = mo.exact_marginals(lat, 1)
        check_f64_against_exact(lat, 0.01, exact)
        frac = mo.tie_fractions(lat)
        assert all(float(frac[n]) == exact[0][n] for n in lat.nodes), s


@pytest.mark.parametrize("ignore_space", [False, True])
def test_exact_pow2(ignore_space):
    """Costs that are multiples of 64 across i16 (homographs, user entries, negative costs) at theta = ln 2 / 64:
    marginals() within one float32 step of the exact value, on sentences of 0-200 characters and one of 1 000."""
    d = adv.make_dictionary("pow2")
    bo = exact_oracle(d, ignore_space)
    theta = math.log(2) / adv.POW2_UNIT
    sents = adv.make_sentences(d, 120, seed=3, max_len=200)
    sents.append(("".join(sents) * 8)[:1000])
    for s in sents:
        if not s.strip(" ") and ignore_space or not s:
            continue
        lat = mo.Lattice(bo, s.encode())
        check_f64_against_exact(lat, theta, mo.exact_marginals(lat, adv.POW2_UNIT, bits=256))


def test_exact_truncated_equals_exact():
    """The 256-bit sums give the same float64 values as the exact ones where the exact ones are affordable."""
    d = adv.make_dictionary("pow2")
    bo = exact_oracle(d)
    sents = [s for s in adv.make_sentences(d, 40, seed=8, max_len=30) if s]
    for s in sents:
        lat = mo.Lattice(bo, s.encode())
        assert mo.exact_marginals(lat, adv.POW2_UNIT) == mo.exact_marginals(lat, adv.POW2_UNIT, bits=256), s


def test_exact_matches_brute_force():
    d = adv.make_dictionary("pow2")
    bo = exact_oracle(d)
    theta = math.log(2) / adv.POW2_UNIT
    for s in [s for s in adv.make_sentences(d, 40, seed=2, max_len=4) if s]:
        lat = mo.Lattice(bo, s.encode())
        prob, pp = mo.exact_marginals(lat, adv.POW2_UNIT)
        bprob, bpp = mo.brute_force(lat, theta)
        assert close(pp, bpp) and all(close(prob[n], bprob[n]) for n in lat.nodes), s


def test_f32_close_refusals():
    exact = [1.0, 0.5, 1e-40]
    mo.assert_f32_close(np.array(exact, dtype=np.float32), exact)
    one_up = np.nextafter(np.float32(0.5), np.float32(1))
    mo.assert_f32_close(np.array([1.0, one_up, 1e-40], dtype=np.float32), exact, ulps=1)
    for bad in ([np.nan, 0.5, 1e-40], [np.inf, 0.5, 1e-40], [-0.0, 0.5, 1e-40], [1.0, 0.5, 1.5e-40], [1.0, 0.5, 0.0]):
        with pytest.raises(AssertionError):
            mo.assert_f32_close(np.array(bad, dtype=np.float32), exact)
    with pytest.raises(AssertionError):
        mo.assert_f32_close(np.array([1.0], dtype=np.float64), [1.0])


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
