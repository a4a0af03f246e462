"""Dictionary and sentences that drive the candidate pool's segment encoding to its limits (test data only).

One dictionary (ids 0..3) serves every fixture:
* char.def: ALPHA (a-z) INVOKE 1 GROUP 1 LENGTH 15, so a run of g <= 15 letters gives exactly g unknown spans and a
  longer one 16; RUN (`Z`) INVOKE 1 GROUP 1 LENGTH 1, one unk.def entry: two candidates per position, one of them
  ending at the end of the run; BIG (`X`) with 70 000 unk.def entries, the cheapest past index 65 535; DEFAULT
  (everything else, INVOKE 0 GROUP 1) for the long user word.
* system lexicon: short words over WORD_LETTERS, keys c^1..c^14 (crowded positions), `QJ`, and 65 535 / 65 536 /
  65 537 homographs of `k` / `l` / `m`, the cheapest one at big_best;
* user lexicon: keys c^1..c^14, 65 537 homographs of `n` (the cheapest at big_best), a word of 4 000 DEFAULT
  characters that starts with the system word `QJ`, and short words over WORD_LETTERS.  (A lexicon field holds at
  most 4 095 bytes, lexicon.rs:124, so no word reaches 32 768 characters on its own: a far lexicon hit needs the
  space skip in front of it.)
`d` is in no key, so a run c^a d^b ends its lexicon hits after a letters while its unknown spans go on."""
import numpy as np

CHAR_DEF = """\
DEFAULT 0 1 0
SPACE 0 1 0
ALPHA 1 1 15
RUN 1 1 1
BIG 1 0 1

0x0020 SPACE
0x0061..0x007A ALPHA
0x005A RUN
0x0058 BIG
"""
WORD_LETTERS = "abefghijoprstuvwy"  # no c, d, k, l, m, n, q, x, z
BIG_UNK = 70000
BIG_UNK_BEST = 69000  # local index of the cheapest BIG entry: past u16
BIG_SYS = {"k": 65535, "l": 65536, "m": 65537}
BIG_USER = ("n", 65537)
BEST_COST = -3000  # the best homograph of a big list: far below the unknown group it competes with
LONG_USER_LEN = 4000
FAR_LEN = 98303
RUN_LEN = 150000
MAX_COUNT = 0xFFFF  # candidates per segment
SPACE_RUN = " " * 40000


def _rows(surface, n, rng, cost_lo=0, cost_hi=400, best=None):
    ids = rng.integers(1, 4, (n, 2))
    costs = rng.integers(cost_lo, cost_hi, n)
    if best is not None:
        costs[best] = BEST_COST
    return [f"{surface},{l},{r},{c},{surface[:8]}{i}" for i, ((l, r), c) in enumerate(zip(ids.tolist(), costs.tolist()))]


def big_best(n):
    """Index of the cheapest homograph of a list of n: the first record of the second segment (65 535) when the
    list splits, else the last record of the only one.  At the start of a sentence that node's row index is the
    same, so it stays within the reference's u16 predecessor index and the best path goes through it: the tokens
    depend on that record being decoded from the right segment."""
    return min(n - 1, MAX_COUNT)


def make_dictionary(seed=0):
    """(lex_csv, matrix, char_def, unk_def, user_csv, long_user_word)"""
    rng = np.random.default_rng([seed, 2024])
    lex = []
    words = set()
    while len(words) < 60:
        words.add("".join(rng.choice(list(WORD_LETTERS), int(rng.integers(1, 4)))))
    for w in sorted(words):
        lex += _rows(w, int(rng.integers(1, 3)), rng)
    lex += _rows("QJ", 1, rng)
    for k in range(1, 15):
        lex += _rows("c" * k, 1, rng, 0, 300)
    for s, n in BIG_SYS.items():
        lex += _rows(s, n, rng, 500, 800, best=big_best(n))
    matrix = "4 4\n" + "".join(f"{r} {l} {int(rng.integers(-20, 21))}\n" for r in range(4) for l in range(4))
    unk = ["DEFAULT,1,1,800,*", "SPACE,0,0,50,*", "ALPHA,1,2,300,*", "RUN,2,3,200,*"]
    big = rng.integers(1000, 1100, BIG_UNK)
    big[BIG_UNK_BEST] = 10
    unk += [f"BIG,3,{1 + i % 3},{int(c)},big{i}" for i, c in enumerate(big.tolist())]
    user = []
    for k in range(1, 15):
        user += _rows("c" * k, 1, rng, 0, 300)
    user += _rows(BIG_USER[0], BIG_USER[1], rng, 500, 800, best=big_best(BIG_USER[1]))
    upper = [chr(c) for c in range(ord("A"), ord("Z")) if chr(c) not in "XZ"]
    long_word = "QJ" + "".join(rng.choice(upper, LONG_USER_LEN - 2))
    user += _rows(long_word, 1, rng, 0, 100)
    uw = set()
    while len(uw) < 15:
        uw.add("".join(rng.choice(list(WORD_LETTERS), int(rng.integers(2, 5)))))
    for w in sorted(uw):
        user += _rows(w, int(rng.integers(1, 3)), rng)
    return "\n".join(lex) + "\n", matrix, CHAR_DEF, "\n".join(unk) + "\n", "\n".join(user) + "\n", long_word


def far_sentences(long_word, seed=0):
    """Sentences over 32 767 characters: end slots far from the slot before them."""
    rng = np.random.default_rng([seed, 7])
    return ["z" * FAR_LEN,
            "".join(rng.choice(list(WORD_LETTERS), FAR_LEN)),  # short system and user words between the far ends
            # with ignore_space the first segment is measured from the space's slot: the user hit needs a move, the
            # system word QJ with the same start comes back 3 998 slots
            SPACE_RUN + long_word + "ab",
            SPACE_RUN + "ab z",
            "Z" * RUN_LEN,
            "ab", ""]


def crowd_sentence(n):
    """c^a d^b followed by a DEFAULT character, whose first position has exactly n segments (unbounded,
    max_grouping_len 0): a user and a system hit per leading c, plus the unknown spans of the a + b letters."""
    for a in range(14, -1, -1):  # as many lexicon hits as the count allows
        for b in range(40):
            g = a + b
            if g and 2 * a + (g if g <= 15 else 16) == n:
                return "c" * a + "d" * b + "-"
    raise ValueError(n)


CROWD_COUNTS = (3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 43, 44)


def crowd_sentences():
    return [crowd_sentence(n) for n in CROWD_COUNTS] + ["ccccccccccccccccccccdddd", "cacdcbc", "cc-ccc ccccccc"]


def big_sentences():
    """Each big source next to one-homograph characters (two adjacent big rows would cost the CPU oracle dearly).  At
    the start of a sentence the best homograph decides the tokens; after a `b` its row index passes u16 and the
    reference's truncated predecessor index decides them."""
    return ["kb", "lb", "mb", BIG_USER[0] + "b", "blb", "b" + BIG_USER[0] + "b", "bXb", "Xa"]


def cut_csv(csv, surface, keep):
    """A lexicon (or unk.def, surface = the category) without the rows of `surface` past its first `keep`."""
    out, seen = [], 0
    for line in csv.splitlines():
        if line.split(",", 1)[0] == surface:
            seen += 1
            if seen > keep:
                continue
        out.append(line)
    return "\n".join(out) + "\n"


# Bounded calls: a boundary that clips a RUN group to exactly 32 767 / 32 768 characters, and one that clips a
# crowded position (c c d^13 -) to 8 / 9 segments.
CLIP_SENTENCE = "Z" * 32770
CLIP_BOUNDS = ([32767], [32768])
CROWD_CLIP_SENTENCE = "cc" + "d" * 13 + "-"
CROWD_CLIP_BOUNDS = ([4], [5])

# Segments outnumber candidates: a batch of RUN groups.  OUTNUMBER_PERMILLE sizes the pool for the candidates but
# not the segments (the CPU tests check it against the model).
OUTNUMBER_SENTENCES = ["Z" * RUN_LEN, "Z" * 5, "", "Z"]
OUTNUMBER_PERMILLE = 2100


def want_cand(n_bytes, permille):
    """engine.cu ensure_workspace: the pool size the estimate gives."""
    return max(1 << 16, int(n_bytes * (permille / 1000.0)) + 4096)
