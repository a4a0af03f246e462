"""Lattice output on the CPU: the restatement (tests/lattice_oracle.py) on a sentence worked by hand, and its
properties over the adversarial dictionaries: the best-path nodes are the C oracle's tokens, every node's cost and
prev follow the `<=` rule of search_min_node, and the node marginals add up to 1 where they must."""
import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
from bounded_oracle import BoundedOracle, wrap
from oracle import vibrato_oracle as vo


def golden_oracle(golden):
    r = golden["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    return od, BoundedOracle(od, r["char.def"], r["unk.def"])


def adversarial_oracle(family, ignore_space=False):
    if family in adv.FAMILIES:
        d, dual = adv.make_dictionary(family), False
    else:
        d, dual = adv.make_dictionary("wrap", dual=family == "dual"), family == "dual"
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=dual)
    od.set_user_csv(d.user_csv)
    return d, od, BoundedOracle(od, d.char_def, d.unk_def, ignore_space)


def test_by_hand(golden):
    """に has two lex.csv rows and nothing else in its lattice: に,2,2,11406 and に,3,3,4481.  From BOS (right id 0)
    matrix.def gives 0->2 = 2124 and 0->3 = 1032, so the nodes cost 2124 + 11406 = 13530 and 1032 + 4481 = 5513; both
    span character 0..1 (bytes 0..3) and follow BOS.  EOS adds 2->0 = -1959 and 3->0 = -2288: the left-id-3 node,
    11571 against 3225 in total, is the best path."""
    od, bo = golden_oracle(golden)
    nodes, links, _ = lo.sentence_lattice(bo, "に".encode())
    assert len(nodes) == 2
    assert sorted(nodes["total_cost"].tolist()) == [5513, 13530]
    for nd in nodes:
        assert (nd["start_char"], nd["end_char"], nd["start_byte"], nd["end_byte"]) == (0, 1, 0, 3)
    assert links["prev"].tolist() == [-1, -1]
    best = nodes[links["flags"] == lo.NODE_BEST]
    assert best["total_cost"].tolist() == [5513] and bo.param(int(best["word_idx"][0]))[0] == 3


def test_by_hand_chain(golden):
    """京都東京都京都 without the user lexicon: every node's prev names a node that ends where it starts, and the
    flagged chain is 京都 / 東京都 / 京都, the C oracle's tokens."""
    od, bo = golden_oracle(golden)
    nodes, links, _ = lo.sentence_lattice(bo, "京都東京都京都".encode())
    for k in range(len(nodes)):
        p = int(links["prev"][k])
        if p < 0:
            assert nodes["start_char"][k] == 0
        else:
            assert nodes["end_char"][p] <= nodes["start_char"][k]
    best = nodes[links["flags"] == lo.NODE_BEST]
    assert best["end_char"].tolist() == [2, 5, 7]
    utf8, off = (np.frombuffer("京都東京都京都".encode(), dtype=np.uint8), np.array([0, 21], dtype=np.uint64))
    _, toks, _ = od.tokenize_batch(utf8, off)
    assert best.tobytes() == toks.tobytes()
    assert np.all(np.diff(nodes["end_char"].astype(np.int64)) >= 0)  # node order: by end position


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
@pytest.mark.parametrize("ignore_space", [False, True])
def test_properties(family, ignore_space):
    d, od, bo = adversarial_oracle(family, ignore_space)
    sents = adv.make_sentences(d, 25, seed=7, max_len=40)
    utf8, off = adv.pack(sents)
    c_off, c_toks, _ = od.tokenize_batch(utf8, off, ignore_space=ignore_space)
    theta = 0.05 if family in adv.FAMILIES else 1e-7
    for i, s in enumerate(sents):
        b = s.encode()
        nodes, links, probs = lo.sentence_lattice(bo, b, theta=theta)
        best = nodes[(links["flags"] & lo.NODE_BEST) != 0]
        exp = c_toks[int(c_off[i]):int(c_off[i + 1])]
        assert best.tobytes() == exp.tobytes(), (family, s)
        if not s:
            assert len(nodes) == 0
            continue
        ends, _, _ = bo.lattice(b, ())
        row_start = {}
        for k in range(len(nodes)):
            row_start.setdefault(int(nodes["end_char"][k]), k)
        for k in range(len(nodes)):
            # the start row of node k, found again from its start_word: the start node is start_word or the start
            # of the skipped space run before it; its min_cost and prev follow the `<=` rule over that row
            e = int(nodes["end_char"][k])
            nd = ends[e][k - row_start[e]]
            left, _, cost = bo.param(nd[2])
            cands = [wrap(l[6] + bo.conn(l[4], left)) for l in ends[nd[0]]]
            m = min(cands)
            pick = max(j for j, v in enumerate(cands) if v == m)
            assert int(nodes["total_cost"][k]) == wrap(m + cost)
            p = int(links["prev"][k])
            if nd[0] == 0:
                assert p == -1
            else:
                assert int(nodes["end_char"][p]) == nd[0] and p - row_start[nd[0]] == (pick & 0xFFFF)
        # the row EOS connects to: its nodes' marginals sum to 1 (row 0, a sentence of skipped spaces, holds only BOS)
        _, (eos_row, _), _ = bo.lattice(b, ())
        assert eos_row == 0 or abs(sum(probs[k] for k in range(len(nodes)) if nodes["end_char"][k] == eos_row) - 1.0) < 1e-9
        if not ignore_space:  # every character lies under exactly one node of every path
            for c in range(len(s)):
                cover = sum(probs[k] for k in range(len(nodes)) if nodes["start_char"][k] <= c < nodes["end_char"][k])
                assert abs(cover - 1.0) < 1e-9, (s, c, cover)


def test_batch_layout(golden):
    od, bo = golden_oracle(golden)
    sents = [b"", "京都".encode(), b"", "に".encode()]
    off, nodes, links, probs = lo.batch_lattice(bo, sents, theta=0.01)
    assert off.tolist()[0] == 0 and off[1] == off[0] and off[3] == off[2] and off[4] - off[3] == 2
    assert len(nodes) == len(links) == len(probs) == int(off[-1])
