"""Seeded dictionaries and sentences for the front end's character classes and UTF-8 input (test data only).

expected_table(char_def) restates CharProperty::from_reader (character.rs:139-216) in plain Python: the base of a
range line is its first category; its id set is the OR of 1 << (id & 31) over the listed categories (the shift of a
release build wraps at 32), OR-ed unmasked into the base's CharInfo, so an id of 18 or more spills into the base id,
INVOKE, GROUP and LENGTH bits; later range lines override earlier ones; a `#` ends a range line's category list.
Code points past the 65 536-entry table take entry 0 (character.rs:112-116).

Families (each a full dictionary: lex.csv, an int16 matrix, unk.def with 1-3 entries for every category, a user
lexicon, all over ALPHABET):
    ``multi``    18 categories, each INVOKE / GROUP pair with each LENGTH of 0, 1, 2 and 15 (all 16 combinations):
                 lines of 2-4 categories, SPACE as a secondary category of letters (x, y, U+FEFF groups with
                 symbols), the pairwise chain p-q-r (p shares with q, q with r, p not with r), U+0000 in a grouping
                 category (so astral characters group with it and with symbols);
    ``wide``     exactly 18 categories, ids 16 and 17 on multi-category lines: two characters that share only bit 17;
    ``spill``    64 categories, so that the secondary ids 18-23 (the base id gains 1 << (id - 18) and lands on another
                 category), 26-31 and 58-63 (INVOKE, GROUP, LENGTH bits), 33 (bit 1: SPACE's) and 50 / 51 (bits 18
                 and 19 again) all exist; no base id reaches the number of categories (ids 24, 25, 56 and 57 would);
    ``refused``  21 categories; one line's secondary id 20 moves base id 17 to 21, which has no unk.def slot.

sentences(family) names each sentence after the edge it reaches: group runs of LENGTH +- 1 and max_grouping_len +
0 / 1 / 2, runs and breaks across characters 31-33 and 511-513 (the 32-character chunks of groupable and
kFrontWarpChars), sentences of 511-513 characters, space runs that group into words, NUL, C0 controls, U+FEFF,
U+FFFF, U+10FFFF and other astral characters.  long_sentence() has more than 16 000 characters (the unpruned Viterbi
twin) and tile_batch() is a 32-sentence tile of more than kFrontStage = 16 384 bytes."""
import numpy as np

FAMILIES = ("multi", "wide", "spill")  # every family a tokenizer accepts
MGLS = (0, 1, 3, 16)  # max_grouping_len values the tests run (0: no limit)
CATE_MASK = (1 << 18) - 1

# 1- to 4-byte characters; every one of them is in some family's char.def or falls to DEFAULT / entry 0
ALPHABET = ["a", "b", "c", "x", "y", "p", "q", "r", "0", "1", "@", " ", "　", "é", "ß", "あ", "い", "ア", "イ",
            "ー", "漢", "字", "\x00", "\x01", "\x1f", "\x7f", "﻿", "￿", "\U00010000", "\U0001F600",
            "\U0010FFFF", "\U00020BB7"]

MULTI_CHAR_DEF = """\
# id: name INVOKE GROUP LENGTH
DEFAULT 0 1 0
SPACE 0 1 0
ALPHA 1 1 0
DIGIT 0 1 1
HIRA 0 0 2
KATA 1 0 15
KANJI 0 1 15
SYM 1 1 2
LINKA 0 1 1
LINKB 1 1 15
NULCAT 1 1 1
LATIN 0 0 0
ND1 0 0 1
ND15 0 0 15
G2 0 1 2
I0 1 0 0
I1 1 0 1
I2 1 0 2

0x0000 NULCAT SYM
0x0001..0x001F SYM
0x0020 SPACE
0x0030..0x0039 DIGIT
0x0040 SYM # KANJI is a comment here
0x0061..0x007A ALPHA
0x0078..0x0079 ALPHA SPACE
0x0070 LINKA
0x0071 LINKB LINKA
0x0072 LINKB
0x007F SYM DEFAULT
0x00DF LATIN
0x00E9 HIRA ALPHA KANJI
0x3000 SPACE KANJI
0x3041..0x3093 HIRA
0x30A1..0x30F6 KATA
0x30FC KATA HIRA SYM DIGIT
0x4E00..0x9FFF KANJI
0xFEFF SPACE SYM
0xFFFF KANJI NULCAT
0x0031 ND1 DIGIT
0x5B57 ND15 KANJI
0x001F G2 SYM
0x30A4 I0 KATA
0x0001 I1
0x007F I2 SYM DEFAULT
"""

WIDE_CHAR_DEF = """\
DEFAULT 0 1 0
SPACE 0 1 0
ALPHA 1 1 0
DIGIT 0 1 1
HIRA 0 0 2
KATA 1 0 15
KANJI 0 1 15
SYM 1 1 2
C8 0 1 1
C9 1 1 0
C10 1 0 3
C11 0 0 1
C12 1 1 4
C13 0 1 0
C14 1 0 0
C15 0 1 2
C16 1 1 0
C17 0 1 3

0x0000 C16 C17
0x0020 SPACE
0x0030..0x0039 DIGIT C16
0x0061..0x007A ALPHA
0x0078 ALPHA SPACE C17
0x0070 C8 C17
0x0071 C13 C17
0x0072 C12 C16 SPACE
0x0040 C15 C16 C17
0x00E9 C10 C11 C17
0x3000 SPACE C16
0x3041..0x3093 HIRA
0x30A1..0x30F6 KATA C9
0x30FC C14 C16
0x4E00..0x9FFF KANJI
0xFEFF SPACE C17
0xFFFF C17
"""

# the spill family's lines over its 64 categories: (code point, [category ids]); unlisted characters are DEFAULT
SPILL_LINES = [
    (0x0000, [7, 33]), (0x0020, [1]), (0x0030, [3, 18]), (0x0031, [3, 19]), (0x0040, [9, 20]), (0x0061, [2, 21]),
    (0x0062, [2, 22]), (0x0063, [2, 23]), (0x0078, [2, 33]), (0x0079, [5, 26]), (0x0070, [4, 27]), (0x0071, [4, 28]),
    (0x0072, [4, 31]), (0x00E9, [6, 58, 59]), (0x00DF, [8, 60, 61, 62]), (0x3000, [1, 63]), (0x3042, [10, 50]),
    (0x3044, [11, 50, 2]), (0x30A2, [12, 29, 30]), (0x30A4, [12, 27]), (0x30FC, [13, 34, 35]), (0x6F22, [14, 27, 18]),
    (0x5B57, [15, 36]), (0x007F, [16, 51]), (0xFEFF, [1, 40, 18]), (0xFFFF, [17, 23, 26]), (0x0001, [39, 44]),
    (0x001F, [45, 20, 27]),
]


def expected_table(char_def, spill=True):
    """(CharInfo of each of the 65 536 table entries, category names by id).  spill=False masks each id set to its 18
    bits before the OR (a wrong restatement, for the tests' mutants)."""
    names, info, ranges = ["DEFAULT"], {}, []
    for line in char_def.splitlines():
        line = line.strip()
        if not line or line.startswith("#"):
            continue
        cols = line.split()
        if not line.startswith("0x"):
            if cols[0] not in names:
                names.append(cols[0])
            i = names.index(cols[0])
            info[i] = (i << 18) | (int(cols[1]) << 26) | (int(cols[2]) << 27) | (int(cols[3]) << 28)
            continue
        lo, _, hi = cols[0].partition("..")
        cats = []
        for c in cols[1:]:
            if c.startswith("#"):
                break
            cats.append(c)
        ranges.append((int(lo, 16), int(hi or lo, 16), cats))

    def encode(cats):
        base = info[names.index(cats[0])]
        idset = base & CATE_MASK
        for c in cats:
            idset |= 1 << (((info[names.index(c)] >> 18) & 0xFF) & 31)
        if not spill:
            idset &= CATE_MASK
        return ((base & ~CATE_MASK) | idset) & 0xFFFFFFFF

    table = [encode(["DEFAULT"])] * 65536
    for lo, hi, cats in ranges:
        v = encode(cats)
        table[lo:hi + 1] = [v] * (hi - lo + 1)
    return table, names


def draw(rng, k):
    """k characters drawn from ALPHABET.  (Not rng.choice(ALPHABET): a numpy string array drops the trailing NUL of
    each element, so U+0000 would come back as the empty string.)"""
    return "".join(ALPHABET[i] for i in rng.integers(0, len(ALPHABET), k))


def char_info(table, cp):
    return table[cp] if cp < len(table) else table[0]


def _spill_char_def(n_cat, lines, seed):
    rng = np.random.default_rng([seed, n_cat])
    names = ["DEFAULT", "SPACE"] + [f"C{i}" for i in range(2, n_cat)]
    out = [f"{n} {int(rng.integers(0, 2))} {int(rng.integers(0, 2))} {int(rng.integers(0, 16))}" for n in names]
    out[0], out[1] = "DEFAULT 0 1 0", "SPACE 0 1 0"
    out.append("")
    out += [f"0x{cp:04X} " + " ".join(names[i] for i in ids) for cp, ids in lines]
    return "\n".join(out) + "\n"


class Family:
    def __init__(self, name, char_def, seed=0):
        self.name = name
        self.char_def = char_def
        self.table, self.categories = expected_table(char_def)
        rng = np.random.default_rng([seed, sum(map(ord, name))])
        n_ids = 8
        surfaces = []
        while len(surfaces) < 60:
            s = draw(rng, int(rng.integers(1, 5)))
            if s not in surfaces and s.strip():
                surfaces.append(s)
        surfaces += ["\x00a", "漢\U0001F600", "\U0010FFFF\x00", "a" * 3, "pq", "ア" * 8]  # NUL and astral surfaces
        self.surfaces = surfaces
        rows = []
        for s in surfaces:
            for _ in range(int(rng.integers(1, 4))):
                l, r = rng.integers(1, n_ids, 2).tolist()
                rows.append(f"{_csv(s)},{l},{r},{int(rng.integers(200, 3000))},w{len(rows)}")
        self.lex_csv = "\n".join(rows) + "\n"
        self.matrix = rng.integers(-50, 51, (n_ids, n_ids)).astype(np.int16)
        unk = []
        for cat in self.categories:
            for _ in range(int(rng.integers(1, 4))):
                l, r = rng.integers(1, n_ids, 2).tolist()
                unk.append(f"{cat},{l},{r},{int(rng.integers(1000, 4000))},unk,{cat}")
        self.unk_def = "\n".join(unk) + "\n"
        user, self.user_surfaces = [], []
        for i in range(12):
            s = surfaces[int(rng.integers(0, len(surfaces)))] + (surfaces[i] if i % 3 == 0 else "")
            l, r = rng.integers(1, n_ids, 2).tolist()
            user.append(f"{_csv(s)},{l},{r},{int(rng.integers(100, 2500))},u{i}")
            self.user_surfaces.append(s)
        self.user_csv = "\n".join(user) + "\n"

    def sources(self):
        """(lex.csv, matrix, char.def, unk.def) for SystemDictionaryBuilder.from_readers / OracleDictionary."""
        return self.lex_csv, self.matrix, self.char_def, self.unk_def

    @property
    def default_info(self):
        """DEFAULT's own CharInfo (what a table without range lines holds everywhere)."""
        return expected_table("\n".join(x for x in self.char_def.splitlines() if not x.startswith("0x")))[0][0]


def _csv(s):
    return f'"{s}"' if any(c in s for c in ',"') else s


def make_family(name, seed=0):
    if name == "multi":
        return Family(name, MULTI_CHAR_DEF, seed)
    if name == "wide":
        return Family(name, WIDE_CHAR_DEF, seed)
    if name == "spill":
        return Family(name, _spill_char_def(64, SPILL_LINES, seed), seed)
    if name == "refused":
        return Family(name, _spill_char_def(21, [(0x0020, [1]), (0x0061, [17, 20]), (0x0062, [3, 18])], seed), seed)
    raise ValueError(name)


def sentences(family):
    """{name: sentence} of the family: the named edges, then 40 seeded random sentences over ALPHABET."""
    s = {}
    for g in (1, 2, 3, 14, 15, 16):  # LENGTH +- 1 of the LENGTH 1 / 2 / 15 classes (DIGIT, SYM, KANJI / KATA)
        s[f"digit_run_{g}"] = "あ" + "0" * g + "あ"
        s[f"sym_run_{g}"] = "い" + "@" * g + "い"
        s[f"kanji_run_{g}"] = "a" + "漢" * g + "a"
        s[f"kata_run_{g}"] = "い" + "ア" * g + "い"
    for m in MGLS[1:]:
        for k in (0, 1, 2):
            s[f"mgl{m}_plus{k}"] = "あ" + "b" * (m + k) + "あ" + "c" * (m + k)
    for e in (31, 32, 33, 511, 512, 513):
        s[f"run_ends_at_{e}"] = "b" * e + "漢" * 3 + "い" * 2
        s[f"run_crosses_{e}"] = "い" * (e - 2) + "abc" + "pqr" + "い"
        s[f"chain_at_{e}"] = "い" * (e - 1) + "pqrpqr" + "い"
        s[f"astral_at_{e}"] = "い" * (e - 1) + "\U0001F600\x00\U0010FFFF@" + "い"
        s[f"space_at_{e}"] = "い" * (e - 1) + "x abc" + "い"
        s[f"len_{e}"] = ("ab漢@x い\U0001F600ー01﻿pqr\x00é" * 40)[:e]
    s["spaces_only"] = "   "
    s["space_run_into_word"] = "xyab  cd"
    s["space_secondary_runs"] = "ab xab yy@@ ﻿@@b 　漢字"
    s["trailing_spaces"] = "abc   "
    s["trailing_grouped_space"] = "漢 xy"
    s["trailing_bom"] = "ab﻿﻿"
    s["leading_space_skip"] = " xabc漢"
    s["nul_inside"] = "ab\x00cd\x00\x00漢"
    s["nul_only"] = "\x00\x00\x00"
    s["controls"] = "\x01\x1f\x7f@\x01a"
    s["specials"] = "a﻿b￿\U0010FFFF\U00010000漢￿"
    s["astral_group"] = "\U0001F600\U00020BB7\x00\U0010FFFF@@a"
    s["multi_cat"] = "éé漢éaー0ーアー@"
    s["chain"] = "pqr rqp pq qr pr"
    # every lexicon word holding NUL or an astral character, so that those words compete with unknown words
    for what, chars in (("nul", "\x00"), ("astral", "\U00010000\U0001F600\U0010FFFF\U00020BB7")):
        words = [w for w in family.surfaces + family.user_surfaces if any(c in w for c in chars)]
        s[f"lexicon_{what}_words"] = "い".join(words)
        s[f"lexicon_{what}_words_joined"] = "".join(words)
    s["flag_combos"] = "11110字字字字\x1f\x1f\x1f@イイイア\x01\x01\x01\x7f\x7f\x7f@ßßß"
    s["one_char"] = "ー"
    s["empty"] = ""
    rng = np.random.default_rng([7, sum(map(ord, family.name))])
    for i in range(40):
        s[f"random_{i}"] = draw(rng, int(rng.integers(1, 60)))
    return s


def long_sentence():
    """More than 16 000 characters: the batch takes the unpruned Viterbi twin."""
    return (("a" * 40 + "pqr" + "漢字" * 3 + "x y" + "\U0001F600" * 3 + "ー" * 5 + "\x00﻿ ") * 260)[:16050]


def tile_batch():
    """32 sentences of 500 characters (each decoded by one warp) holding more than kFrontStage bytes of text in one
    k_front tile, which then reads its text from global memory."""
    rng = np.random.default_rng(11)
    return [draw(rng, 500) for _ in range(32)]


CONTINUATIONS = (0x00, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xFF)


def utf8_cases():
    """Every 1- and 2-byte string; every lead byte 0x80-0xFF followed by 1-3 of CONTINUATIONS; each of those cut
    short at the end of the sentence (after an `a`)."""
    out = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    seqs = []
    for lead in range(0x80, 0x100):
        for c1 in CONTINUATIONS:
            seqs.append(bytes([lead, c1]))
            for c2 in CONTINUATIONS:
                seqs.append(bytes([lead, c1, c2]))
                for c3 in CONTINUATIONS:
                    seqs.append(bytes([lead, c1, c2, c3]))
    out += seqs
    out += [b"a" + s[:k] for s in seqs if len(s) > 2 for k in range(1, len(s))]
    return out
