"""Character classes and UTF-8 validity on the CPU: the char.def fixtures of tests/charclass_fixtures.py read by the
host dictionary, the oracle and a plain restatement; the bounded oracle's lattice against the C oracle on every
fixture sentence; and a mutant restatement per edge, each of which must change a token on the fixtures' sentences
(so that the GPU tests built on the same sentences would see that slip in a kernel)."""
import numpy as np
import pytest

import charclass_fixtures as cf
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo

HIGH_CODE_POINTS = [0x10000, 0x1F600, 0x20BB7, 0x10FFFF]


def dictionaries(f):
    od = vo.OracleDictionary(*f.sources())
    od.set_user_csv(f.user_csv)
    return od


def encoded(f, with_long=False):
    sents = list(cf.sentences(f).values()) + ([cf.long_sentence()] if with_long else [])
    return [s.encode() for s in sents]


def oracle_tokens(od, sents, isp, mgl):
    utf8, off = vb.Tokenizer.pack(sents)
    return od.tokenize_batch(utf8, off, isp, mgl)[:2]


def test_spill_family_reaches_its_ids():
    """The spill family's lines name the ids they are meant to reach, and no base id leaves the categories."""
    f = cf.make_family("spill")
    ids = {i for _, line in cf.SPILL_LINES for i in line[1:]}
    assert set(range(18, 24)) <= ids and set(range(26, 32)) <= ids and set(range(58, 64)) <= ids and 33 in ids
    assert len(f.categories) == 64 and max((v >> 18) & 0xFF for v in f.table) < 64
    assert len(cf.make_family("wide").categories) == 18
    refused = cf.make_family("refused")
    assert max((v >> 18) & 0xFF for v in refused.table) == len(refused.categories)


def test_multi_family_flag_combinations():
    """multi holds every INVOKE / GROUP pair with every LENGTH of 0, 1, 2 and 15, each on a character of ALPHABET."""
    f = cf.make_family("multi")
    got = {((v >> 26) & 1, (v >> 27) & 1, v >> 28) for v in (cf.char_info(f.table, ord(c)) for c in cf.ALPHABET)}
    assert got >= {(i, g, n) for i in (0, 1) for g in (0, 1) for n in (0, 1, 2, 15)}


@pytest.mark.parametrize("family", cf.FAMILIES)
def test_nul_and_astral_words_reach_the_sentences(family):
    """Every lexicon word (system and user) holding NUL or an astral character occurs in a fixture sentence, the random
    sentences and the large tile hold NUL, and the oracle's best paths take lexicon words holding NUL and astral
    characters, so that the GPU tests see those characters complete a lexicon match."""
    f = cf.make_family(family)
    sents = cf.sentences(f)
    words = [w for w in f.surfaces + f.user_surfaces if "\x00" in w or any(ord(c) > 0xFFFF for c in w)]
    assert any("\x00" in w for w in words) and any(any(ord(c) > 0xFFFF for c in w) for w in words)
    for w in words:
        assert any(w in s for s in sents.values()), repr(w)
    assert any("\x00" in s for k, s in sents.items() if k.startswith("random_"))
    assert all(len(s) == 500 for s in cf.tile_batch()) and any("\x00" in s for s in cf.tile_batch())
    od = dictionaries(f)
    utf8, off = vb.Tokenizer.pack(list(sents.values()))
    tok_off, toks, _ = od.tokenize_batch(utf8, off)
    buf = bytes(utf8)
    won = set()  # surfaces of the lexicon words on the best paths
    for i in range(len(off) - 1):
        for t in toks[int(tok_off[i]):int(tok_off[i + 1])]:
            if int(t["word_idx"]) >> 30 != 2:
                won.add(buf[int(off[i]) + int(t["start_byte"]):int(off[i]) + int(t["end_byte"])].decode())
    assert any("\x00" in w for w in won) and any(any(ord(c) > 0xFFFF for c in w) for w in won)


@pytest.mark.parametrize("family", cf.FAMILIES + ("refused",))
def test_tables_agree(family):
    """Dictionary.char_info, OracleDictionary.char_info and the restatement agree on every code point
    0..0x10FFFF, before and after a .dic write and read.  The oracle refuses `refused` (see below)."""
    f = cf.make_family(family)
    d = vb.SystemDictionaryBuilder.from_readers(*f.sources())
    d2 = vb.Dictionary.read(d.write())
    od = dictionaries(f) if family != "refused" else None
    table = f.table
    for cp in range(0x110000):
        e = table[cp] if cp < 65536 else table[0]
        assert d.char_info(cp) == e, hex(cp)
        if od is not None:
            assert od.char_info(cp) == e, hex(cp)
        if cp < 65536 or cp in HIGH_CODE_POINTS:
            assert d2.char_info(cp) == e, hex(cp)


def test_oracle_refuses_base_without_unk_slot():
    """A spill that moves a base id to the number of categories: the oracle refuses the dictionary with the device
    image's message instead of indexing unk.def out of bounds; so does the device image after a .dic round trip."""
    f = cf.make_family("refused")
    with pytest.raises(vo.OracleError, match="CharInfo base_id has no unk.def slot"):
        vo.OracleDictionary(*f.sources())
    d = vb.SystemDictionaryBuilder.from_readers(*f.sources())
    for dic in (d, vb.Dictionary.read(d.write())):
        with pytest.raises(vb.VibratoError, match="CharInfo base_id has no unk.def slot") as ei:
            dic.pack_blob()
        assert ei.value.kind == "BincodeDecode"


@pytest.mark.parametrize("family", cf.FAMILIES)
def test_restatement_matches_oracle(family):
    """BoundedOracle (the restatement the GPU tests compare with) equals the C oracle on every fixture sentence,
    with and without ignore_space, at every max_grouping_len."""
    f = cf.make_family(family)
    od = dictionaries(f)
    sents = encoded(f)
    for isp in (False, True):
        for mgl in cf.MGLS:
            tok_off, toks = oracle_tokens(od, sents, isp, mgl)
            got_off, got = BoundedOracle(od, f.char_def, f.unk_def, isp, mgl).tokenize_batch(sents)
            np.testing.assert_array_equal(got_off, tok_off)
            assert got.tobytes() == toks.tobytes(), (isp, mgl)


def test_restatement_long_sentence():
    """The sentence of more than 16 000 characters, once."""
    f = cf.make_family("multi")
    od = dictionaries(f)
    sents = [cf.long_sentence().encode()]
    tok_off, toks = oracle_tokens(od, sents, True, 3)
    got_off, got = BoundedOracle(od, f.char_def, f.unk_def, True, 3).tokenize_batch(sents)
    assert got.tobytes() == toks.tobytes()


# ---- mutants: each restates one plausible slip of the front end ----

class BaseBitOnly(BoundedOracle):
    """The id set reduced to the base category's bit: secondary categories never group."""
    def char_infos(self, text):
        return [(c & ~cf.CATE_MASK) | ((1 << ((c >> 18) & 31)) & cf.CATE_MASK) for c in super().char_infos(text)]


class CommonCategory(BoundedOracle):
    """Transitive grouping: a run holds while one category bit is common to all of its characters."""
    @staticmethod
    def groupable(ci):
        n, grp = len(ci), []
        for i in range(n):
            acc, j = ci[i] & cf.CATE_MASK, i
            while j + 1 < n and acc & ci[j + 1]:
                acc &= ci[j + 1]
                j += 1
            grp.append(j - i + 1)
        return grp


class NoChunkCarry(BoundedOracle):
    """groupable solved per 32-character chunk without the carry from the chunk to its right."""
    @staticmethod
    def groupable(ci):
        return [min(g, 32 - i % 32) for i, g in enumerate(BoundedOracle.groupable(ci))]


class AstralDefault(BoundedOracle):
    """Code points past the table take DEFAULT's CharInfo instead of entry 0's."""
    default = 0

    def char_infos(self, text):
        return [self.default if ord(ch) > 0xFFFF else c for ch, c in zip(text, super().char_infos(text))]


class LengthThreeBits(BoundedOracle):
    """LENGTH read through a 3-bit mask."""
    def char_infos(self, text):
        return [c & ~(1 << 31) for c in super().char_infos(text)]


class Mask17(BoundedOracle):
    """The id-set mask of groupable one bit short: category 17 never groups."""
    @staticmethod
    def groupable(ci):
        return BoundedOracle.groupable([c & 0x1FFFF for c in ci])


class NoSpill(BoundedOracle):
    """Category ids of 18 and more masked away instead of spilling into the base id and flag bits."""
    table = None

    def char_infos(self, text):
        return [cf.char_info(self.table, ord(ch)) for ch in text]


class BaseSpaceOnly(BoundedOracle):
    """The space skip tested on the base category only."""
    def skips(self, c):
        return bool(self.space_mask) and (1 << ((c >> 18) & 0xFF)) == self.space_mask


class NulEndsText(BoundedOracle):
    """NUL taken as the end of the text."""
    def lattice(self, sent, bounds, trace=None):
        return super().lattice(sent.split(b"\0")[0], bounds, trace)


class StrictMaxGrouping(BoundedOracle):
    """`g - 1 < max_grouping_len` in place of `<=` (for a limit of 2 or more, the true rule at the limit minus one)."""
    def __init__(self, od, char_def, unk_def, ignore_space=False, max_grouping_len=0):
        super().__init__(od, char_def, unk_def, ignore_space, max_grouping_len - 1)


def _no_spill(f):
    NoSpill.table = cf.expected_table(f.char_def, spill=False)[0]


def _astral(f):
    AstralDefault.default = f.default_info


# mutant, the families and (ignore_space, max_grouping_len) settings to look in, a setup hook
MUTANTS = [
    (BaseBitOnly, ("multi",), ((False, 0),), None),
    (CommonCategory, ("multi",), ((False, 0),), None),
    (NoChunkCarry, ("multi",), ((False, 0),), None),
    (AstralDefault, ("multi",), ((False, 0),), _astral),
    (LengthThreeBits, ("multi",), ((False, 0),), None),
    (Mask17, ("wide",), ((False, 0),), None),
    (NoSpill, ("spill",), ((False, 0), (True, 0)), _no_spill),
    (BaseSpaceOnly, ("multi", "wide", "spill"), ((True, 0),), None),
    (NulEndsText, ("multi",), ((False, 0),), None),
    (StrictMaxGrouping, ("multi",), ((False, 3), (False, 16)), None),
]


@pytest.mark.parametrize("mutant,families,settings,setup", MUTANTS, ids=[m[0].__name__ for m in MUTANTS])
def test_mutant_is_killed(mutant, families, settings, setup):
    """Each mutant changes at least one token of the fixture sentences it names; the sentence that shows it is
    reported, so a fixture that stops reaching its edge fails here rather than silently in the GPU tests."""
    for fam in families:
        f = cf.make_family(fam)
        od = dictionaries(f)
        if setup:
            setup(f)
        named = cf.sentences(f)
        for isp, mgl in settings:
            m = mutant(od, f.char_def, f.unk_def, isp, mgl)
            for name, s in named.items():
                b = s.encode()
                _, exp = oracle_tokens(od, [b], isp, mgl)
                if m.tokenize(b).tobytes() != exp.tobytes():
                    print(f"{mutant.__name__} killed by {fam}:{name} (ignore_space={isp}, max_grouping_len={mgl})")
                    return
    pytest.fail(f"no fixture sentence tells {mutant.__name__} from the oracle")


# ---- UTF-8 validity ----

def python_valid(b):
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def test_utf8_valid_matches_python():
    cases = cf.utf8_cases()
    assert len(cases) > 200000
    bad = [c for c in cases if vo.utf8_valid(c) != python_valid(c)]
    assert not bad, [c.hex() for c in bad[:10]]
