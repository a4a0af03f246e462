"""Segmentation sampling on the CPU: Philox4x32-10 against its known answers, and the sampling restatement
(tests/sampling_oracle.py) against the exact path distribution of tests/marginal_oracle.py."""
import math
from collections import Counter

import pytest
from scipy import stats

import adversarial as adv
import marginal_oracle as mo
import sampling_oracle as so
from test_marginal_oracle import adversarial_oracle, golden_oracle


@pytest.mark.parametrize("ctr, key, out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, out):
    assert so.philox4x32_10(ctr, key) == out


def test_uniform_bits():
    """u takes 27 + 26 bits of the first two words and lies in [0, 1)."""
    x = so.philox4x32_10((3, 1, 7, 0), (5, 0))
    assert so.uniform(5, 3, 1, 7) == ((x[0] >> 5) * 2.0 ** 26 + (x[1] >> 6)) / 2.0 ** 53
    us = [so.uniform(2 ** 64 - 1, t, 0, 0) for t in range(1000)]
    assert all(0.0 <= u < 1.0 for u in us) and 0.4 < sum(us) / len(us) < 0.6


def _chi_square(lat, theta, draws, seed):
    """p-value of the oracle's path frequencies against P(path) over `draws` samples of sentence 0."""
    paths = mo.all_paths(lat)
    cmin = min(c for c, _ in paths)
    weights = [math.exp(-theta * (c - cmin)) for c, _ in paths]
    z = sum(weights)
    index = {tuple(p): k for k, (_, p) in enumerate(paths)}
    fw = so.forward(lat, theta)
    counts = Counter()
    for j in range(draws):
        path, _ = so.walk(lat, fw, theta, seed, 0, j)
        counts[index[tuple(path)]] += 1
    expected = [draws * w / z for w in weights]
    # pool the paths too rare for the chi-square approximation into one cell
    big = [k for k, e in enumerate(expected) if e >= 5]
    small = [k for k in range(len(paths)) if k not in big]
    obs = [counts[k] for k in big] + ([sum(counts[k] for k in small)] if small else [])
    exp = [expected[k] for k in big] + ([sum(expected[k] for k in small)] if small else [])
    assert sum(counts.values()) == draws and len(obs) >= 2
    return stats.chisquare(obs, exp).pvalue


@pytest.mark.parametrize("sent, theta", [("に", 0.0002), ("京都東京都京都", 0.001), ("東京都", 0.002),
                                         ("東京都京都", 0.001)])
def test_frequencies_match_path_probabilities(golden, sent, theta):
    bo = golden_oracle(golden)
    lat = mo.Lattice(bo, sent.encode())
    assert _chi_square(lat, theta, 4000, seed=12345) > 1e-4


@pytest.mark.parametrize("family", ["ties", "flat_columns"])
def test_frequencies_adversarial(family):
    d, bo = adversarial_oracle(family)
    sents = [s for s in adv.make_sentences(d, 40, seed=3, max_len=6) if s]
    tested = 0
    for s in sents:
        lat = mo.Lattice(bo, s.encode())
        n_paths = len(mo.all_paths(lat))
        if not 3 <= n_paths <= 60:
            continue
        assert _chi_square(lat, 0.05, 3000, seed=99) > 1e-4, s
        tested += 1
        if tested == 3:
            break
    assert tested


def test_prefix_costs_and_best_path(golden):
    """Every sample's records carry the wrapped prefix costs of its own path; a sample on the best path equals the
    tokens byte for byte."""
    bo = golden_oracle(golden)
    for sent in ["京都東京都京都", "東京都に行った。", "kampersanda"]:
        b = sent.encode()
        tokens = bo.tokenize(b)
        lat = mo.Lattice(bo, b)
        best = lat.best_path()
        for rec, path, _ in so.sentence_samples(bo, b, 64, 0.001, 7, 0):
            assert rec["total_cost"][-1] == so.wrap32(so.path_cost(lat, path) - lat.w(path[-1], None))
            if path == best:
                assert rec.tobytes() == tokens.tobytes()


@pytest.mark.parametrize("family", ["ties", "flat_columns"])
def test_large_theta_tie_fractions(family):
    """At large theta every sample is a minimum-cost path, and a node is sampled as often as its share of them."""
    d, bo = adversarial_oracle(family)
    sents = [s for s in adv.make_sentences(d, 40, seed=9, max_len=30) if s]
    draws, seen_fraction = 400, False
    for s in sents[:12]:
        lat = mo.Lattice(bo, s.encode())
        frac = mo.tie_fractions(lat)
        fw = so.forward(lat, 100.0)
        cmin = fw[2]  # R(EOS): the least exact cost
        counts = Counter()
        for j in range(draws):
            path, _ = so.walk(lat, fw, 100.0, 1, 0, j)
            assert so.path_cost(lat, path) == cmin
            counts.update(path)
        for n in lat.nodes[1:]:
            f = float(frac[n])
            if f == 0:
                assert counts[n] == 0, (s, n)
            else:
                sd = math.sqrt(draws * f * (1 - f)) + 1e-9
                assert abs(counts[n] - draws * f) <= 5 * sd + 1, (s, n, counts[n], f)
            seen_fraction |= 0 < f < 1
    assert seen_fraction


def test_empty_and_deterministic(golden):
    bo = golden_oracle(golden)
    assert [len(r) for r, _, _ in so.sentence_samples(bo, b"", 3, 1.0, 0, 0)] == [0, 0, 0]
    a = so.sentence_samples(bo, "京都東京都京都".encode(), 5, 0.001, 2 ** 64 - 1, 17)
    b = so.sentence_samples(bo, "京都東京都京都".encode(), 5, 0.001, 2 ** 64 - 1, 17)
    assert [x[1] for x in a] == [x[1] for x in b]
