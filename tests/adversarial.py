"""Seeded adversarial dictionaries and corpora for the Viterbi kernels (test data only, MeCab-format text).

The synthetic dictionaries of vibrato_b200.synth draw costs from wide normal distributions, so two path totals are
almost never equal and the rules that decide ties never decide a token.  These dictionaries are built so that they
do, on every route k_viterbi / k_viterbi2 can take:

* a small alphabet (1-, 2-, 3- and 4-byte UTF-8, one astral character) and many 1-4 character surfaces with 1-40
  homographs each, plus a user lexicon over the same surfaces: lattice rows longer than k_viterbi2's 32-entry
  staging pass, and positions with more candidates than one warp holds;
* char.def / unk.def with INVOKE, GROUP and LENGTH set on part of the alphabet, so unknown words join the ties;
* cost families:
    ``ties``          matrix in {-1, 0, 1}, word costs in {0, 1, 2};
    ``flat_columns``  M[r][l] = c_l: every connection into l costs exactly its lower bound lb[l], so the pruning
                      test of a tying predecessor is decided at equality;
    ``extreme``       matrix and word costs from {-32768, -32767, -1, 0, 1, 32766, 32767}; some columns all 32767
                      (the bound prunes hard), others holding -32768 (nothing is pruned);
    ``wrap``          Raw / Dual connector: bigram.cost values near +-2^31, so template sums wrap in i32 and the
                      Dual connector's matrix part hits its i16 clamp.

Two more dictionaries have marginals that are exact rationals (tests/marginal_oracle.exact_marginals):
    ``pow2``          matrix and word costs from POW2, multiples of 64 across the i16 range: at theta = ln 2 / 64
                      every path weighs a power of two;
    zero_dictionary() every cost 0: a node's marginal is a ratio of path counts, at any theta.
"""
import numpy as np

# a, b, é (2 bytes), あ, ア, 漢 (3 bytes), 1, 𠮷 (4 bytes, astral; DEFAULT class)
ALPHABET = ["a", "b", "é", "あ", "ア", "漢", "1", "\U00020bb7"]
FAMILIES = ("ties", "flat_columns", "extreme")
EXTREME = np.array([-32768, -32767, -1, 0, 1, 32766, 32767], dtype=np.int64)
POW2 = np.array([-32768, -32704, -4096, -64, 0, 64, 128, 4096, 32704], dtype=np.int64)  # all multiples of 64
POW2_UNIT = 64
WRAP_COSTS = np.array([2147483647, 2147480000, -2147483648, -2147480000, 1 << 30, -(1 << 30), 0, 1, -1], dtype=np.int64)
N_IDS = 10  # connection ids 0..9 (0 = BOS/EOS)

CHAR_DEF = """\
DEFAULT 0 1 0
SPACE 0 1 0
ALPHA 1 1 0
HIRAGANA 0 1 2
KATAKANA 1 1 2
KANJI 0 0 2
NUMERIC 1 0 3

0x0020 SPACE
0x0061..0x0062 ALPHA
0x00E9 ALPHA
0x3042 HIRAGANA
0x30A2 KATAKANA
0x6F22 KANJI
0x0031 NUMERIC
"""
CATEGORIES = ["DEFAULT", "SPACE", "ALPHA", "HIRAGANA", "KATAKANA", "KANJI", "NUMERIC"]


class AdversarialDictionary:
    """Sources of one adversarial dictionary: `matrix` is an int16 ndarray [num_left, num_right] (data[left *
    num_right + right]) or, for the ``wrap`` family, the tuple (bigram.right, bigram.left, bigram.cost)."""

    def __init__(self, family, lex_csv, matrix, unk_def, user_csv, surfaces, homographs):
        self.family = family
        self.lex_csv = lex_csv
        self.matrix = matrix
        self.char_def = CHAR_DEF
        self.unk_def = unk_def
        self.user_csv = user_csv
        self.surfaces = surfaces  # distinct system surfaces, in generation order
        self.homographs = homographs  # system rows per surface


def _word_costs(family, rng, n):
    if family in ("extreme", "wrap"):
        return rng.choice(EXTREME, n)
    if family == "pow2":
        return rng.choice(POW2, n)
    return rng.integers(0, 3, n)


def _matrix(family, rng):
    """int16 [num_left, num_right]; column l of the issue's M[r][l] notation is row l here."""
    if family == "pow2":
        return rng.choice(POW2, (N_IDS, N_IDS)).astype(np.int16)
    if family == "ties":
        return rng.integers(-1, 2, (N_IDS, N_IDS)).astype(np.int16)
    if family == "flat_columns":
        return np.repeat(rng.integers(-3, 4, (N_IDS, 1)), N_IDS, axis=1).astype(np.int16)
    m = rng.choice(EXTREME, (N_IDS, N_IDS))
    m[rng.permutation(np.arange(1, N_IDS))[:3]] = 32767  # the bound prunes every predecessor but the cheapest
    for l in range(N_IDS):
        if l % 3 == 0:
            m[l, int(rng.integers(0, N_IDS))] = -32768  # lb[l] = -32768: nothing is pruned
    return m.astype(np.int16)


def _bigram_files(rng, n_templates):
    """bigram.right / bigram.left / bigram.cost over ids 1..N_IDS-1: three feature values per template, a cost for
    every (right, left) value pair of every template, drawn near +-2^31."""
    def feats(side):
        rows = []
        for i in range(1, N_IDS):
            cols = ["*" if rng.random() < 0.15 else f"{side}{t}:v{int(rng.integers(0, 3))}" for t in range(n_templates)]
            rows.append(f"{i}\t" + ",".join(cols))
        return "\n".join(rows) + "\n"
    right, left = feats("R"), feats("L")
    costs = [f"R{t}:v{a}/L{t}:v{b}\t{int(rng.choice(WRAP_COSTS))}" for t in range(n_templates) for a in range(3) for b in range(3)]
    return right, left, "\n".join(costs) + "\n"


def make_dictionary(family, seed=0, n_surfaces=70, dual=False):
    """family in FAMILIES, "pow2", or "wrap" (Raw connector; `dual` picks the Dual connector's 10 templates)."""
    assert family in FAMILIES + ("wrap", "pow2")
    fam = FAMILIES.index(family) if family in FAMILIES else {"wrap": 9, "pow2": 10}[family]
    rng = np.random.default_rng([seed, fam, int(dual)])
    surfaces = []
    while len(surfaces) < n_surfaces:
        s = "".join(rng.choice(ALPHABET, int(rng.integers(1, 5))))
        if s not in surfaces:
            surfaces.append(s)
    # 1-40 homographs: mostly few, a tail past 32 (a row longer than one staging pass of k_viterbi2)
    homographs = np.minimum(rng.geometric(0.12, n_surfaces), 40)
    homographs[: 4] = [40, 36, 33, 40]
    rows = []
    for s, h in zip(surfaces, homographs.tolist()):
        ids = rng.integers(1, N_IDS, (h, 2))
        for (l, r), c in zip(ids.tolist(), _word_costs(family, rng, h).tolist()):
            rows.append(f"{s},{l},{r},{c},w{len(rows)}")
    lex_csv = "\n".join(rows) + "\n"
    if family == "wrap":
        matrix = _bigram_files(rng, 10 if dual else 4)
    else:
        matrix = _matrix(family, rng)
    unk = []
    for cat in CATEGORIES:
        n = int(rng.integers(1, 4))
        for (l, r), c in zip(rng.integers(1, N_IDS, (n, 2)).tolist(), _word_costs(family, rng, n).tolist()):
            unk.append(f"{cat},{l},{r},{c},unk,{cat}")
    unk_def = "\n".join(unk) + "\n"
    user = []
    for i in range(25):  # homographs of system surfaces, and compounds of two of them
        s = surfaces[int(rng.integers(0, n_surfaces))]
        if i % 3 == 0:
            s += surfaces[int(rng.integers(0, n_surfaces))]
        for (l, r), c in zip(rng.integers(1, N_IDS, (int(rng.integers(1, 6)), 2)).tolist(), _word_costs(family, rng, 5).tolist()):
            user.append(f"{s},{l},{r},{c},u{len(user)}")
    user_csv = "\n".join(user) + "\n"
    return AdversarialDictionary(family, lex_csv, matrix, unk_def, user_csv, surfaces, homographs)


ZERO_CHAR_DEF = """\
DEFAULT 0 1 0
SPACE 0 1 0
ALPHA 0 0 0
BEE 1 1 2

0x0020 SPACE
0x0061 ALPHA
0x0062 BEE
"""


def zero_dictionary():
    """Every word and connection cost 0: the surfaces a, aa and aaa (a sentence of n `a` has T(n) paths, the
    tribonacci numbers, about 1.84^n), unknown words of `b` (grouped, and of 1 and 2 characters) and of every other
    character; no user lexicon (user_csv is empty).  The marginals are ratios of path counts at any theta."""
    lex = "a,1,1,0,A\naa,1,1,0,AA\naaa,1,1,0,AAA\n"
    matrix = np.zeros((2, 2), dtype=np.int16)
    unk = "DEFAULT,1,1,0,unk\nSPACE,1,1,0,space\nALPHA,1,1,0,alpha\nBEE,1,1,0,bee\n"
    d = AdversarialDictionary("zero", lex, matrix, unk, "", ["a", "aa", "aaa", "b"], [1, 1, 1, 0])
    d.char_def = ZERO_CHAR_DEF
    return d


def make_sentences(d, n_sent, seed=1, max_len=300):
    """Sentences of 0-`max_len` characters (log-uniform): dictionary surfaces, single characters and space runs,
    cut at the drawn length; about 3% are empty and 8% end in a run of spaces."""
    rng = np.random.default_rng([seed, 77])
    lens = np.floor(np.exp(rng.uniform(0, np.log(max_len + 1), n_sent))).astype(np.int64)
    lens[rng.random(n_sent) < 0.03] = 0
    out = []
    for n in lens.tolist():
        parts, have = [], 0
        while have < n:
            r = rng.random()
            if r < 0.7:
                p = d.surfaces[int(rng.integers(0, len(d.surfaces)))]
            elif r < 0.9:
                p = str(rng.choice(ALPHABET))
            else:
                p = " " * int(rng.integers(1, 4))
            parts.append(p)
            have += len(p)
        s = "".join(parts)[:n]
        if n and rng.random() < 0.08:
            k = int(rng.integers(1, min(n, 3) + 1))
            s = s[: n - k] + " " * k
        out.append(s)
    return out


def pack(sentences):
    """list[str] -> (utf8 uint8[], byte_offsets uint64[n + 1])"""
    blobs = [s.encode("utf-8") for s in sentences]
    off = np.zeros(len(blobs) + 1, dtype=np.uint64)
    if blobs:
        off[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
    return np.frombuffer(b"".join(blobs), dtype=np.uint8), off


def single_word_dictionary(w, c, with_aa=None):
    """One word `a` of cost w, a 1 x 1 matrix holding c, char.def INVOKE 0: the lattice of "a" * n has one path,
    whose k-th node (1-based) costs wrap_i32(k * (w + c)).  `with_aa` adds a word `aa` of that cost, so that the
    search compares wrapped totals."""
    lex = f"a,0,0,{w},A\n" + (f"aa,0,0,{with_aa},AA\n" if with_aa is not None else "")
    matrix = f"1 1\n0 0 {c}\n"
    char_def = "DEFAULT 0 1 0\nSPACE 0 1 0\n0x0020 SPACE\n"
    unk_def = "DEFAULT,0,0,0,unk\nSPACE,0,0,0,space\n"
    return lex, matrix, char_def, unk_def


def wrap_i32(x):
    return (int(x) + (1 << 31)) % (1 << 32) - (1 << 31)


def threshold_dictionary(seed=0):
    """The ``ties`` dictionary plus a word `z` (three homographs, cost -32768) on a connection id S whose every
    connection on the all-`z` path (BOS -> z, z -> z, z -> EOS) costs -32768: a sentence of n `z` ends at
    n * -65536 - 32768, about -1.05e9 for n = 16 000 — the largest magnitude k_viterbi2's pruned arithmetic admits."""
    d = make_dictionary("ties", seed)
    S = N_IDS
    m = np.zeros((N_IDS + 1, N_IDS + 1), dtype=np.int16)
    m[:N_IDS, :N_IDS] = d.matrix
    m[S, :] = -32768  # into z from anything (BOS included)
    m[0, S] = -32768  # z -> EOS
    d.matrix = m
    d.lex_csv += "".join(f"z,{S},{S},-32768,z{i}\n" for i in range(3))
    return d
