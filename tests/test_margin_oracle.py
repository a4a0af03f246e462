"""Near-best lattices on the CPU: the restatement (tests/margin_oracle.py) against a brute-force enumeration of every
BOS -> EOS path, and the guarantees of the option "lattice_margin" (include/vibrato_b200.h) over golden and
adversarial sentences, required boundaries and required tokens."""
import json
import os

import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import margin_oracle as mgo
import marginal_oracle as mo
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_TEXTS = ["京都東京都京都", "東京都に行った", "abcdefgh", "東京   都", "一橋大学大学院", "に", "kampersanda"]


def golden_oracle(user=True, ignore_space=False, cls=BoundedOracle):
    with open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8") as f:
        r = json.load(f)["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        od.set_user_csv(r["user.csv"])
    return cls(od, r["char.def"], r["unk.def"], ignore_space)


def adversarial_oracle(family, ignore_space=False):
    d = adv.make_dictionary(family)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od.set_user_csv(d.user_csv)
    return d, BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


def brute(lat):
    """(per node: least cost of a path through it, best) from every path."""
    paths = mo.all_paths(lat)
    through = {}
    for cost, nodes in paths:
        for n in nodes:
            through[n] = min(through.get(n, cost), cost)
    return through, min((c for c, _ in paths), default=None)


def cases():
    out = [("golden", golden_oracle(), [t.encode() for t in GOLDEN_TEXTS])]
    out.append(("golden_space", golden_oracle(ignore_space=True), [t.encode() for t in GOLDEN_TEXTS]))
    for fam in adv.FAMILIES:  # "ties" has tens of homographs per row: its short sentences have 10^5 paths
        d, bo = adversarial_oracle(fam, ignore_space=fam == "ties")
        out.append((fam, bo, [s.encode() for s in adv.make_sentences(d, 14, seed=5, max_len=3 if fam == "ties" else 6)]))
    return out


@pytest.mark.parametrize("name,bo,texts", cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_margins_are_the_brute_force_ones(name, bo, texts):
    """margin(n) = (least cost of a path through n) - best, for every node on some path; no margin elsewhere."""
    checked = 0
    for t in texts:
        if not t:
            continue
        lat = mo.Lattice(bo, t)
        mg, best = mgo.margins(lat)
        through, b2 = brute(lat)
        assert best == b2, t
        assert mg == {n: c - best for n, c in through.items()}, t
        assert min(mg.values(), default=0) == 0
        checked += len(mg)
    assert checked > 20


def union_within(lat, D):
    paths = mo.all_paths(lat)
    if not paths:
        return set()
    best = min(c for c, _ in paths)
    return {n for c, nodes in paths if c <= best + D for n in nodes}


@pytest.mark.parametrize("name,bo,texts", cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_guarantees(name, bo, texts):
    """Path closure for several D, D = 0 (the union of the minimum-cost paths), D = 2^62 (every node with a path to
    EOS), the best path always kept, and the remapped links."""
    for t in texts:
        if not t:
            assert len(mgo.pruned_lattice(bo, t, 0)[0]) == 0
            continue
        lat = mo.Lattice(bo, t)
        mg, best = mgo.margins(lat)
        pos = sorted(set(mg.values()))
        for D in sorted({0, 1, 500, 5000, mgo.MAX_MARGIN} | set(pos[:3])):
            kept = mgo.kept_nodes(lat, D, lat.best_path())
            assert kept == union_within(lat, D), (t, D)
            if D == mgo.MAX_MARGIN:
                assert kept == set(mg)
            nodes, links, margins, _ = mgo.pruned_lattice(bo, t, D)
            full_nodes, full_links, _ = lo.sentence_lattice(bo, t)
            assert len(nodes) == len(kept) and np.all(margins <= D) and np.all(margins >= 0)
            best_full = full_nodes[(full_links["flags"] & lo.NODE_BEST) != 0]
            assert nodes[(links["flags"] & lo.NODE_BEST) != 0].tobytes() == best_full.tobytes()
            # without i32 wrap a kept node's predecessor is kept: no -2 link
            assert np.all(links["prev"] >= -1), (t, D)
            for k in range(len(nodes)):
                p = int(links["prev"][k])
                assert (p == -1) == (nodes["start_char"][k] == 0 or p == -1)
                if p >= 0:
                    assert nodes["end_char"][p] <= nodes["start_char"][k] and margins[p] <= margins[k]


def test_bounds_and_spans():
    """The restatement runs unchanged over BoundedOracle's boundaries and SpanOracle's required tokens."""
    so = golden_oracle(cls=SpanOracle)
    checked = 0
    for text, cons in [("京都東京都京都", Constraints((6,), ())), ("京都東京都京都", Constraints((), ((6, 15, None),))),
                       ("東京都に行った", Constraints((), ((0, 6, "名詞"),))), ("abcdefgh", Constraints((3, 5), ()))]:
        lat = mo.Lattice(so, text.encode(), cons)
        mg, best = mgo.margins(lat)
        through, b2 = brute(lat)
        assert best == b2 and mg == {n: c - best for n, c in through.items()}
        for D in (0, 700, mgo.MAX_MARGIN):
            assert mgo.kept_nodes(lat, D, lat.best_path()) == union_within(lat, D)
            nodes, links, margins, _ = mgo.pruned_lattice(so, text.encode(), D, cons)
            checked += len(nodes)
    assert checked > 10


def test_wrapping_costs_keep_the_best_path():
    """Where i32 costs wrap the tokenizer's best path is not the least exact cost: its nodes are kept, with margin > 0."""
    files = adv.single_word_dictionary(-32768, -32768, with_aa=0)
    bo = BoundedOracle(vo.OracleDictionary(*files), files[2], files[3])
    t = ("a" * 33000).encode()
    nodes, links, margins, _ = mgo.pruned_lattice(bo, t, 0)
    best = (links["flags"] & lo.NODE_BEST) != 0
    full_nodes, full_links, _ = lo.sentence_lattice(bo, t)
    assert nodes[best].tobytes() == full_nodes[(full_links["flags"] & lo.NODE_BEST) != 0].tobytes()
    assert margins[best].max() > 0 and margins[~best].max() == 0
