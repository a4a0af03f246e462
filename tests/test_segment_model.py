"""The segment model (tests/segment_model.py) on the fixtures of tests/test_gpu_segments.py: decoding gives back every
position's candidates, and each fixture reaches the edge of the encoding it is there for.  Runs without a GPU."""
import pytest

import segment_fixtures as sf
import segment_model as sm
from adversarial import pack
from bounded_oracle import BoundedOracle, vo_dictionary


@pytest.fixture(scope="module")
def dic():
    lex, matrix, char_def, unk_def, user, long_word = sf.make_dictionary()
    od = vo_dictionary(lex, matrix, char_def, unk_def, user)
    return od, long_word, {isp: BoundedOracle(od, char_def, unk_def, isp) for isp in (False, True)}, unk_def


def seg_counts(enc):
    return [c for _, _, c in sm.walk(0, enc)]


def unk_words(bo, cat):
    return [(2 << 30) | (w & 0xFFFF) for w in range(bo.unk_off[cat], bo.unk_off[cat + 1])]


ALPHA, RUN = 2, 3


def check_roundtrip(pos, stride=1):
    for slot in sorted(pos)[::stride]:
        cands = pos[slot]
        enc = sm.encode(slot, cands)
        assert [sm.cand_at(slot, enc, j) for j in range(len(cands))] == cands, slot
        assert all(abs(d) <= sm.MAX_DELTA for d in sm.deltas(enc))


def first_delta(pos, slot):
    segs = sm.encode(slot, pos[slot])
    return sm.deltas(segs)[0], sm.moves(segs)


@pytest.mark.parametrize("mgl", [0, 3, 20])
def test_closed_form_runs_equal_the_oracle(dic, mgl):
    """unknown_cands / run_positions, which stand in for BoundedOracle on the long runs, equal its trace on short ones."""
    od, _, _, unk_def = dic
    bo = BoundedOracle(od, sf.CHAR_DEF, unk_def, False, mgl)
    for ch, cat, length in (("z", ALPHA, 15), ("Z", RUN, 1)):
        for n in list(range(1, 24)) + [40]:
            assert sm.positions(bo, (ch * n).encode()) == sm.run_positions(n, length, unk_words(bo, cat), mgl), (ch, n)


def test_far_ends(dic):
    _, long_word, bos, _ = dic
    bo = bos[False]
    run = sm.run_positions(sf.RUN_LEN, 1, unk_words(bo, RUN))
    far = sm.run_positions(sf.FAR_LEN, 15, unk_words(bo, ALPHA))
    check_roundtrip(run, 7)
    check_roundtrip(far, 61)

    def at(pos, n, r):  # the position with r characters left in its run
        return n - r

    # first segment: the grouped span, delta r
    assert first_delta(run, at(run, sf.RUN_LEN, 32767)) == (32767, 0)
    assert first_delta(run, at(run, sf.RUN_LEN, 32768)) == (32767, 1)  # a move, then 1
    assert first_delta(far, at(far, sf.FAR_LEN, 32768)) == (32767, 1)
    # second source: the span of length 1, delta 1 - r
    for pos, n in ((run, sf.RUN_LEN), (far, sf.FAR_LEN)):
        s = at(pos, n, 32768)
        segs = sm.encode(s, pos[s])
        assert sm.deltas(segs)[:3] == [32767, 1, -32767] and sm.moves(segs) == 1  # -32 767: no move
        s = at(pos, n, 32769)
        segs = sm.encode(s, pos[s])
        assert sm.deltas(segs)[:4] == [32767, 2, -32767, -1] and sm.moves(segs) == 2  # -32 768: one move
        s = at(pos, n, 65536)
        segs = sm.encode(s, pos[s])
        assert sm.deltas(segs)[:6] == [32767, 32767, 2, -32767, -32767, -1] and sm.moves(segs) == 4  # past +-65 534
    assert max(sm.moves(sm.encode(s, c)) for s, c in far.items()) >= 4
    # ignore_space: the first segment is measured from the space's slot.  The user word of 4 000 characters behind
    # 40 000 spaces needs a move of the user kind, the system word QJ with the same start a negative delta.
    n = len(sf.SPACE_RUN)
    pos = sm.positions(bos[True], (sf.SPACE_RUN + long_word + "ab").encode())
    check_roundtrip(pos)
    segs = sm.encode(0, pos[0])
    assert [k for k, _, _ in sm.walk(0, segs)[:3]] == [1, 1, 0]  # user (a move, then the hit), then system
    assert sm.deltas(segs)[:3] == [32767, n + sf.LONG_USER_LEN - 32767, 2 - sf.LONG_USER_LEN]
    pos = sm.positions(bos[True], (sf.SPACE_RUN + "ab z").encode())
    check_roundtrip(pos)
    d, mv = first_delta(pos, 0)
    assert (d, mv) == (32767, 1) and pos[0][0][0] > n


def test_bounded_clips(dic):
    od, _, bos, _ = dic
    bo = bos[False]
    got = []
    for bounds in sf.CLIP_BOUNDS:
        pos = sm.positions(bo, sf.CLIP_SENTENCE.encode(), bounds)
        check_roundtrip(pos)
        got.append(first_delta(pos, 0))
    assert got == [(32767, 0), (32767, 1)]  # a group clipped to 32 767 / 32 768 characters
    counts = []
    for bounds in sf.CROWD_CLIP_BOUNDS:
        pos = sm.positions(bo, sf.CROWD_CLIP_SENTENCE.encode(), bounds)
        check_roundtrip(pos)
        counts.append(sm.n_segments(sm.encode(0, pos[0])))
    assert counts == [8, 9]


def test_big_sources(dic):
    """The big lists split as the encoder must split them, and each big source decides its sentence's tokens: cut
    to the records before its cheapest one (the first record of the second segment, or the last of a 65 535 list;
    the first segment of the unk.def category), the C oracle
    tokenizes the sentence differently.  So a GPU route that decoded a later segment's records wrongly, or lost the
    user kind in the split, could not give the oracle's tokens."""
    od, _, bos, _ = dic
    bo = bos[False]
    sizes = {}
    for s in sf.big_sentences():
        pos = sm.positions(bo, s.encode())
        check_roundtrip(pos)
        for slot, cands in pos.items():
            for lt, end, words in sm.sources(cands):
                if len(words) > 1000:
                    runs = [c for k, e, c in sm.walk(slot, sm.encode(slot, cands)) if (k, e) == (lt, end) and c]
                    sizes[(lt, len(words))] = runs
    assert sizes == {(0, 65535): [65535], (0, 65536): [65535, 1], (0, 65537): [65535, 2], (1, 65537): [65535, 2],
                     (2, sf.BIG_UNK): [65535, sf.BIG_UNK - 65535]}
    lex, matrix, char_def, unk_def, user, _ = sf.make_dictionary()
    cuts = {**{k: ("sys", k, sf.big_best(n)) for k, n in sf.BIG_SYS.items()},  # keep the records before the best
            sf.BIG_USER[0]: ("user", sf.BIG_USER[0], sf.big_best(sf.BIG_USER[1])), "X": ("unk", "BIG", sf.MAX_COUNT)}
    for s in sf.big_sentences():
        big = [c for c in s if c in cuts]
        assert len(big) == 1, s
        where, surface, keep = cuts[big[0]]
        cut = {"sys": lex, "user": user, "unk": unk_def}[where]
        cut = sf.cut_csv(cut, surface, keep)
        od_cut = vo_dictionary(cut if where == "sys" else lex, matrix, char_def, cut if where == "unk" else unk_def,
                               cut if where == "user" else user)
        utf8, off = pack([s])
        full = od.tokenize_batch(utf8, off)[1]
        part = od_cut.tokenize_batch(utf8, off)[1]
        assert full.tobytes() != part.tobytes(), s
        assert full.tobytes() == bo.tokenize(s.encode()).tobytes(), s


def test_crowded_positions(dic):
    od, _, bos, _ = dic
    bo = bos[False]
    seen = set()
    for n, s in zip(sf.CROWD_COUNTS, sf.crowd_sentences()):
        pos = sm.positions(bo, s.encode())
        check_roundtrip(pos)
        enc = sm.encode(0, pos[0])
        assert sm.n_segments(enc) == n, s
        assert {k for k, _, _ in sm.walk(0, enc)} == {0, 1, 2}, s  # user, system and unknown segments mixed
    for s in sf.crowd_sentences():
        pos = sm.positions(bo, s.encode())
        seen |= {sm.n_segments(sm.encode(slot, c)) for slot, c in pos.items()}
    for g in (4, 8, 16, 32):
        assert {g - 1, g, g + 1} <= seen
    assert {7, 8, 9} <= seen and max(seen) >= 33
    assert all(len(s.encode()) <= 16000 for s in sf.crowd_sentences() + sf.big_sentences())


def test_segments_outnumber_candidates(dic):
    """The batch of RUN groups has nearly 3x more segments than candidates, and OUTNUMBER_PERMILLE sizes the pool
    between the two, so only the segments overflow it."""
    od, _, bos, _ = dic
    words = unk_words(bos[False], RUN)
    pos, slot = {}, 0
    for s in sf.OUTNUMBER_SENTENCES:
        pos.update(sm.run_positions(len(s), 1, words, slot0=slot))
        slot += len(s) + 1
    segs, cands = sm.totals(pos)
    assert segs > 2.5 * cands
    n_bytes = sum(len(s) for s in sf.OUTNUMBER_SENTENCES)
    assert cands < sf.want_cand(n_bytes, sf.OUTNUMBER_PERMILLE) < segs
    # the long sentence alone in a chunk (the chunked pipeline sizes from the largest chunk)
    long_pos = sm.run_positions(sf.RUN_LEN, 1, words)
    s1, c1 = sm.totals(long_pos)
    assert c1 < sf.want_cand(sf.RUN_LEN, sf.OUTNUMBER_PERMILLE) < s1
