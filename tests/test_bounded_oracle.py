"""Required token boundaries (vbt_tokenize_batch_bounded) on the CPU: hand-worked cases on the golden fixture and
properties of the bounded oracle (tests/bounded_oracle.py) over the adversarial dictionaries.  The oracle is checked
against the C restatement where no boundary is given."""
import numpy as np
import pytest

import adversarial as adv
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo


def golden_oracle(golden, user=False, ignore_space=False, mgl=0):
    r = golden["resources"]
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        od.set_user_csv(r["user.csv"])
    return BoundedOracle(od, r["char.def"], r["unk.def"], ignore_space, mgl)


def surfaces(sent, toks):
    b = sent.encode()
    return [b[t["start_byte"]:t["end_byte"]].decode() for t in toks]


def lex_types(toks):
    return [int(t["word_idx"]) >> 30 for t in toks]


def matrix_cost(golden, right, left):
    for line in golden["resources"]["matrix.def"].splitlines()[1:]:
        r, l, c = map(int, line.split())
        if (r, l) == (right, left):
            return c
    raise KeyError((right, left))


@pytest.mark.parametrize("user", [False, True])
def test_boundary_rules_out_tokyo_to(golden, user):
    """京都|東京|都京都: a boundary after 東京 (byte 12) rules out 東京都 (and the user word 京都東京都).  The cheapest
    remaining path is 京都 東京 都 京都 (lex.csv ids 6/6, 6/6, 8/8, 6/6), whose cost is the sum of the word costs and
    matrix.def connections written out below."""
    s = "京都東京都京都"
    bo = golden_oracle(golden, user=user)
    toks = bo.tokenize(s.encode(), [12])
    assert surfaces(s, toks) == ["京都", "東京", "都", "京都"]
    assert lex_types(toks) == [0, 0, 0, 0]
    c = lambda r, l: matrix_cost(golden, r, l)  # noqa: E731
    expected = []
    total = 0
    for word_cost, (right_prev, left) in [(5293, (0, 6)), (2816, (6, 6)), (2914, (6, 8)), (5293, (8, 6))]:
        total += c(right_prev, left) + word_cost
        expected.append(total)
    assert [int(t["total_cost"]) for t in toks] == expected
    assert [int(t["start_char"]) for t in toks] == [0, 2, 4, 5]
    unb = bo.tokenize(s.encode())
    assert "東京都" in surfaces(s, unb) or "京都東京都" in surfaces(s, unb)


def test_boundary_splits_a_character_group(golden):
    """ALPHA groups (char.def GROUP 1, LENGTH 0): a boundary inside the run clips the group on both sides."""
    bo = golden_oracle(golden)
    s = "abcdef"
    assert surfaces(s, bo.tokenize(s.encode())) == ["abcdef"]
    toks = bo.tokenize(s.encode(), [3])
    assert surfaces(s, toks) == ["abc", "def"]
    assert lex_types(toks) == [2, 2]


def test_boundary_admits_a_group_max_grouping_len_rejected(golden):
    """max_grouping_len 3: from positions 0-3 of an 8-letter run the group is too long (more than 3 further
    characters) and LENGTH 0 leaves only the one-character fallback, so only "efgh" groups; a boundary after "abcd"
    makes the group at position 0 short enough."""
    bo = golden_oracle(golden, mgl=3)
    s = "abcdefgh"
    assert surfaces(s, bo.tokenize(s.encode())) == ["a", "b", "c", "d", "efgh"]
    assert surfaces(s, bo.tokenize(s.encode(), [4])) == ["abcd", "efgh"]


def test_boundary_inside_skipped_spaces(golden):
    """ignore_space: a boundary inside a skipped run of spaces holds trivially; the tokens do not change."""
    bo = golden_oracle(golden, ignore_space=True)
    s = "東京   都"
    toks = bo.tokenize(s.encode(), [7])
    assert surfaces(s, toks) == ["東京", "都"]
    assert [(int(t["start_byte"]), int(t["end_byte"])) for t in toks] == [(0, 6), (9, 12)]
    np.testing.assert_array_equal(toks, bo.tokenize(s.encode()))


def adversarial_oracles():
    for fam in list(adv.FAMILIES) + ["raw", "dual"]:
        if fam in adv.FAMILIES:
            d, dual = adv.make_dictionary(fam), False
        else:
            d, dual = adv.make_dictionary("wrap", dual=fam == "dual"), fam == "dual"
        od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=dual)
        od.set_user_csv(d.user_csv)
        yield fam, d, od


def lead_bytes(b):
    return [i for i in range(len(b) + 1) if i == len(b) or (b[i] & 0xC0) != 0x80]


def random_bounds(rng, b, k):
    return sorted(int(x) for x in rng.choice(lead_bytes(b), size=min(k, len(lead_bytes(b))), replace=False))


@pytest.mark.parametrize("ignore_space", [False, True])
def test_properties_over_adversarial_dictionaries(ignore_space):
    rng = np.random.default_rng(7)
    for fam, d, od in adversarial_oracles():
        bo = BoundedOracle(od, d.char_def, d.unk_def, ignore_space)
        sents = adv.make_sentences(d, 40, seed=5, max_len=60) + [" a ", "あ ア  ", ""]
        utf8, off = adv.pack(sents)
        c_off, c_toks = od.tokenize_batch(utf8, off, ignore_space, 0)[:2]
        p_off, p_toks = bo.tokenize_batch([s.encode() for s in sents])
        np.testing.assert_array_equal(c_off, p_off)
        np.testing.assert_array_equal(c_toks, p_toks.astype(c_toks.dtype))
        for i, s in enumerate(sents):
            b = s.encode()
            base = p_toks[int(p_off[i]):int(p_off[i + 1])]
            # empty lists and lists of only 0 / len give the unbounded tokens
            np.testing.assert_array_equal(bo.tokenize(b, []), base)
            np.testing.assert_array_equal(bo.tokenize(b, [0, 0, len(b)]), base)
            # no token crosses a boundary (random, with duplicates)
            bnd = random_bounds(rng, b, 3)
            bnd = sorted(bnd + bnd[:1])
            for t in bo.tokenize(b, bnd):
                assert not any(t["start_byte"] < x < t["end_byte"] for x in bnd), (fam, s, bnd)
            # the unbounded path's own boundaries keep it in the constrained lattice, which can only gain candidates
            # (lexicon words past a boundary no longer suppress unknown words): its cost does not rise.  Costs that
            # wrap around i32 (the raw / dual bigram costs) are not ordered, so only the Matrix families are compared.
            own = sorted({int(t["start_byte"]) for t in base} | {int(t["end_byte"]) for t in base})
            if fam in adv.FAMILIES:
                assert bo.best_cost(b, own) <= bo.best_cost(b), (fam, s)
            # a boundary at every character: one-character tokens only
            every = lead_bytes(b)
            assert all(t["end_char"] - t["start_char"] == 1 for t in bo.tokenize(b, every)), (fam, s)
