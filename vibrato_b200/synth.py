"""Seeded synthetic MeCab-format dictionaries and Japanese-like corpora (numpy only).

No real ipadic / unidic dictionary exists in this environment (no network), so the benchmark
configurations of BASELINE.json are concretised with shape-matched synthetic data as laid out in
SURVEY.md §8(d):

  * ``synth-ipadic``  — 392 126 words, 1316 x 1316 connection matrix (ipadic-mecab-2.7.0's shape)
  * ``synth-unidic``  — 876 803 words, 15 388 x 15 626 matrix = 459 MiB (unidic-cwj-3.1.1's shape)
  * ``synth-tiny``    — a few thousand words, for fast tests

Every report that uses these must say "synthetic".  The generators are deterministic in `seed`.
"""
import numpy as np

# MeCab-style character classes (category INVOKE GROUP LENGTH, then code-point ranges).
CHAR_DEF = """\
DEFAULT 0 1 0
SPACE 0 1 0
KANJI 0 0 2
SYMBOL 1 1 0
NUMERIC 1 1 0
ALPHA 1 1 0
HIRAGANA 0 1 2
KATAKANA 1 1 2
KANJINUMERIC 1 1 0
GREEK 1 1 0
CYRILLIC 1 1 0

0x0020 SPACE
0x00D0 SPACE
0x0009 SPACE
0x000B SPACE
0x000A SPACE

0x0021..0x002F SYMBOL
0x0030..0x0039 NUMERIC
0x003A..0x0040 SYMBOL
0x0041..0x005A ALPHA
0x005B..0x0060 SYMBOL
0x0061..0x007A ALPHA
0x007B..0x007E SYMBOL

0x00A1..0x00BF SYMBOL
0x00C0..0x00FF ALPHA
0x0100..0x017F ALPHA
0x0374..0x03FB GREEK
0x0400..0x04F9 CYRILLIC

0x3000 SPACE
0x3001..0x303F SYMBOL
0x3041..0x309F HIRAGANA
0x30A1..0x30FF KATAKANA
0x31F0..0x31FF KATAKANA
0x30FC KATAKANA

0x3400..0x4DB5 KANJI
0x4E00..0x9FA5 KANJI
0xF900..0xFA2D KANJI

0x4E00 KANJINUMERIC KANJI
0x4E8C KANJINUMERIC KANJI
0x4E09 KANJINUMERIC KANJI
0x56DB KANJINUMERIC KANJI
0x4E94 KANJINUMERIC KANJI
0x516D KANJINUMERIC KANJI
0x4E03 KANJINUMERIC KANJI
0x516B KANJINUMERIC KANJI
0x4E5D KANJINUMERIC KANJI
0x5341 KANJINUMERIC KANJI
0x767E KANJINUMERIC KANJI
0x5343 KANJINUMERIC KANJI
0x4E07 KANJINUMERIC KANJI
0x5104 KANJINUMERIC KANJI
0x5146 KANJINUMERIC KANJI

0xFF10..0xFF19 NUMERIC
0xFF21..0xFF3A ALPHA
0xFF41..0xFF5A ALPHA
0xFF66..0xFF9D KATAKANA
0xFF9E..0xFF9F KATAKANA
"""

UNK_CATEGORIES = ["DEFAULT", "SPACE", "KANJI", "SYMBOL", "NUMERIC", "ALPHA", "HIRAGANA", "KATAKANA",
                  "KANJINUMERIC", "GREEK", "CYRILLIC"]

SHAPES = {
    # name: (n_words, num_right, num_left, homograph_mean, n_kanji)
    "synth-tiny": (4000, 64, 72, 1.3, 400),
    "synth-small": (40000, 400, 410, 1.3, 1500),
    "synth-ipadic": (392126, 1316, 1316, 1.3, 4000),
    "synth-unidic": (876803, 15388, 15626, 2.2, 5000),
}

HIRAGANA = np.arange(0x3041, 0x3094, dtype=np.uint32)
KATAKANA = np.concatenate([np.arange(0x30A1, 0x30F7, dtype=np.uint32), np.array([0x30FC], dtype=np.uint32)])
ASCII_ALPHA = np.concatenate([np.arange(0x61, 0x7B, dtype=np.uint32), np.arange(0x41, 0x5B, dtype=np.uint32)])
DIGITS = np.arange(0x30, 0x3A, dtype=np.uint32)
PUNCT = np.array([0x3001, 0x3002, 0x300C, 0x300D, 0x30FB, 0x21, 0x3F, 0x2C, 0x2E, 0xFF01, 0xFF1F], dtype=np.uint32)


def _kanji_alphabet(n):
    # common-use block first; deterministic stride so neighbours are not all adjacent code points
    base = 0x4E00 + (np.arange(n, dtype=np.uint64) * 37) % (0x9FA5 - 0x4E00)
    return np.unique(base.astype(np.uint32))


def _zipf_choice(rng, n_items, size, s=1.0):
    """Zipf(s) over ranks 0..n_items-1 by inverse-CDF (exact, vectorised)."""
    w = 1.0 / np.power(np.arange(1, n_items + 1, dtype=np.float64), s)
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    return np.searchsorted(cdf, rng.random(size), side="left").astype(np.int64)


def encode_utf8(cps):
    """Vectorised UTF-8 encoding of a uint32 code-point array -> (bytes uint8[], byte length per char)."""
    cps = np.asarray(cps, dtype=np.uint32)
    nb = np.where(cps < 0x80, 1, np.where(cps < 0x800, 2, np.where(cps < 0x10000, 3, 4))).astype(np.int64)
    start = np.zeros(len(cps) + 1, dtype=np.int64)
    np.cumsum(nb, out=start[1:])
    out = np.zeros(int(start[-1]), dtype=np.uint8)
    s = start[:-1]
    m1 = nb == 1
    out[s[m1]] = cps[m1]
    m2 = nb == 2
    out[s[m2]] = 0xC0 | (cps[m2] >> 6)
    out[s[m2] + 1] = 0x80 | (cps[m2] & 0x3F)
    m3 = nb == 3
    out[s[m3]] = 0xE0 | (cps[m3] >> 12)
    out[s[m3] + 1] = 0x80 | ((cps[m3] >> 6) & 0x3F)
    out[s[m3] + 2] = 0x80 | (cps[m3] & 0x3F)
    m4 = nb == 4
    out[s[m4]] = 0xF0 | (cps[m4] >> 18)
    out[s[m4] + 1] = 0x80 | ((cps[m4] >> 12) & 0x3F)
    out[s[m4] + 2] = 0x80 | ((cps[m4] >> 6) & 0x3F)
    out[s[m4] + 3] = 0x80 | (cps[m4] & 0x3F)
    return out, start


class SynthDictionary:
    """MeCab-format sources of a synthetic dictionary plus the surface table used to draw corpora."""

    def __init__(self, name, lex_csv, matrix, char_def, unk_def, surf_cps, surf_off, kanji, shape):
        self.name = name
        self._shape = shape  # (num_left, num_right)
        self.lex_csv = lex_csv  # bytes
        self.matrix = matrix  # int16 [num_left, num_right]  (data[left * num_right + right])
        self.char_def = char_def  # str
        self.unk_def = unk_def  # str
        self.surf_cps = surf_cps  # uint32 flat code points of the distinct surfaces
        self.surf_off = surf_off  # int64 [n_surfaces + 1]
        self.kanji = kanji

    @property
    def num_left(self):
        return self._shape[0]

    @property
    def num_right(self):
        return self._shape[1]

    def matrix_def(self):
        """Text matrix.def (only sensible for small shapes)."""
        nl, nr = self.matrix.shape
        lines = [f"{nr} {nl}"]
        for l in range(nl):
            row = self.matrix[l]
            lines.extend(f"{r} {l} {int(row[r])}" for r in range(nr))
        return "\n".join(lines) + "\n"


def make_dictionary(name="synth-tiny", seed=20260923, with_matrix=True):
    """`with_matrix=False` skips the (large) connection matrix and unk.def: enough to draw corpora."""
    n_words, num_right, num_left, homo_mean, n_kanji = SHAPES[name]
    rng = np.random.default_rng(seed)
    kanji = _kanji_alphabet(n_kanji)
    n_surf = int(n_words / homo_mean)

    # --- distinct surfaces: length geometric (mean 2.6) clipped to 1..8; script mix per word ---
    lens = np.minimum(rng.geometric(1 / 2.6, size=int(n_surf * 1.6)), 8).astype(np.int64)
    script = rng.choice(4, size=len(lens), p=[0.42, 0.40, 0.12, 0.06])  # hira / kanji(+okurigana) / kata / ascii
    total = int(lens.sum())
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    word_of = np.repeat(np.arange(len(lens)), lens)
    pos_in = np.arange(total) - off[:-1][word_of]
    sc = script[word_of]
    cps = np.empty(total, dtype=np.uint32)
    r = rng.random(total)
    # hiragana words: Zipf-ish over kana so that short kana strings collide a lot (dense lattice)
    hz = _zipf_choice(rng, len(HIRAGANA), total, 0.8)
    kz = _zipf_choice(rng, len(kanji), total, 0.9)
    tz = _zipf_choice(rng, len(KATAKANA), total, 0.5)
    az = rng.integers(0, len(ASCII_ALPHA), total)
    cps[:] = HIRAGANA[hz]
    mk = sc == 1
    # kanji words: kanji stem, trailing chars may be okurigana (hiragana) with p=0.35 beyond the first
    use_kanji = mk & ((pos_in == 0) | (r > 0.35))
    cps[use_kanji] = kanji[kz[use_kanji]]
    mt = sc == 2
    cps[mt] = KATAKANA[tz[mt]]
    ma = sc == 3
    cps[ma] = ASCII_ALPHA[az[ma]]
    # dedupe surfaces, keep first n_surf distinct (order = generation order => frequent shapes first)
    keys = {}
    cl = cps.tolist()
    ol = off.tolist()
    order = []
    for i in range(len(lens)):
        k = tuple(cl[ol[i]:ol[i + 1]])
        if k not in keys:
            keys[k] = len(order)
            order.append(k)
            if len(order) >= n_surf:
                break
    # guarantee every kana and frequent kanji exists as a 1-char word (like real dictionaries)
    for c in HIRAGANA.tolist() + KATAKANA.tolist() + kanji[: n_kanji // 2].tolist():
        k = (c,)
        if k not in keys:
            keys[k] = len(order)
            order.append(k)
    n_surf = len(order)
    surf_len = np.array([len(k) for k in order], dtype=np.int64)
    surf_off = np.zeros(n_surf + 1, dtype=np.int64)
    np.cumsum(surf_len, out=surf_off[1:])
    surf_cps = np.fromiter((c for k in order for c in k), dtype=np.uint32, count=int(surf_off[-1]))

    # --- rows: each surface gets 1 + geometric homographs until n_words rows; shuffled row order ---
    mult = rng.geometric(1.0 / homo_mean, size=n_surf).astype(np.int64)
    row_surf = np.repeat(np.arange(n_surf), mult)
    if len(row_surf) < n_words:
        extra = rng.integers(0, n_surf, n_words - len(row_surf))
        row_surf = np.concatenate([row_surf, extra])
    rng.shuffle(row_surf)
    row_surf = row_surf[:n_words]
    # make sure every surface keeps at least one row (so the corpus sampler only draws real words)
    left = _zipf_choice(rng, num_left - 1, n_words, 1.0) + 1
    right = _zipf_choice(rng, num_right - 1, n_words, 1.0) + 1
    lperm = rng.permutation(num_left - 1)
    rperm = rng.permutation(num_right - 1)
    left = lperm[left - 1] + 1  # ids are not frequency sorted in a raw dictionary
    right = rperm[right - 1] + 1
    cost = np.clip(np.rint(rng.normal(6000, 2500, n_words)), -32768, 32767).astype(np.int64)
    surf_strs = ["".join(map(chr, k)) for k in order]
    rs = row_surf.tolist()
    ll, rl, cc = left.tolist(), right.tolist(), cost.tolist()
    pos_names = ["名詞,普通名詞,一般", "動詞,一般,*", "助詞,格助詞,*", "形容詞,一般,*", "副詞,*,*", "名詞,固有名詞,地名"]
    lines = []
    for i in range(n_words):
        s = surf_strs[rs[i]]
        lines.append(f"{s},{ll[i]},{rl[i]},{cc[i]},{pos_names[i % 6]},*,*,{s},{s},w{i}")
    # a few rows that exercise the CSV corner cases: quoted surface with a comma, quoted feature
    lines.append('"１,２",3,3,4000,名詞,数詞,"a,b",*')
    lines.append("、,1,1,2000,補助記号,読点,*,*,*,*")
    lines.append("。,2,2,1500,補助記号,句点,*,*,*,*")
    lex_csv = ("\n".join(lines) + "\n").encode("utf-8")

    # --- connection matrix ~ N(0, 1500^2); row/col 0 (BOS/EOS) milder ---
    if not with_matrix:
        return SynthDictionary(name, lex_csv, None, CHAR_DEF, None, surf_cps, surf_off, kanji, (num_left, num_right))
    matrix = np.empty((num_left, num_right), dtype=np.int16)
    chunk = max(1, (1 << 24) // num_right)
    for s in range(0, num_left, chunk):
        e = min(num_left, s + chunk)
        matrix[s:e] = np.clip(np.rint(rng.standard_normal((e - s, num_right), dtype=np.float32) * 1500.0),
                              -32768, 32767).astype(np.int16)
    matrix[0, :] = (matrix[0, :] // 4).astype(np.int16)
    matrix[:, 0] = (matrix[:, 0] // 4).astype(np.int16)

    # --- unk.def: 4-6 entries per category ---
    ulines = []
    for ci, cat in enumerate(UNK_CATEGORIES):
        for j in range(4 + (ci % 3)):
            ulines.append(f"{cat},{int(rng.integers(1, num_left))},{int(rng.integers(1, num_right))},"
                          f"{int(rng.integers(3000, 15000))},名詞,未知語,{cat},{j}")
    unk_def = "\n".join(ulines) + "\n"
    return SynthDictionary(name, lex_csv, matrix, CHAR_DEF, unk_def, surf_cps, surf_off, kanji, (num_left, num_right))


def make_user_csv(d, n_rows=1000, seed=20260927):
    """User lexicon (config 4): some rows overlap system surfaces, some are new compounds, some cheap."""
    rng = np.random.default_rng(seed)
    n_surf = len(d.surf_off) - 1
    rows = []
    for i in range(n_rows):
        a = int(rng.integers(0, min(n_surf, 5000)))
        k = d.surf_cps[d.surf_off[a]:d.surf_off[a + 1]].tolist()
        if i % 3 != 0:  # compound of two system words
            b = int(rng.integers(0, min(n_surf, 5000)))
            k = k + d.surf_cps[d.surf_off[b]:d.surf_off[b + 1]].tolist()
        s = "".join(map(chr, k))
        cost = int(rng.integers(-3000, 6000))
        rows.append(f"{s},{int(rng.integers(1, d.num_left))},{int(rng.integers(1, d.num_right))},{cost},ユーザー名詞,u{i}")
    return ("\n".join(rows) + "\n").encode("utf-8")


def make_corpus(d, n_sent, seed=20260924, mean_len=40.0, sd_len=8.0, min_len=8, max_len=120, fixed_len=None,
                log_uniform=None, unk_frac=0.05, space_frac=0.01, astral_frac=0.001, user_csv=None, user_frac=0.0):
    """Sentences as (utf8 uint8[], offsets uint64[n_sent+1]).

    Text = dictionary surfaces drawn Zipf(1.0) by surface rank, concatenated into one stream and cut
    at the per-sentence lengths (so cuts may fall inside a word); `unk_frac` of the drawn items are
    replaced by out-of-dictionary runs (ASCII, digits, rare kanji, katakana), `space_frac` by spaces.
    """
    rng = np.random.default_rng(seed)
    if fixed_len is not None:
        lens = np.full(n_sent, int(fixed_len), dtype=np.int64)
    elif log_uniform is not None:
        lo, hi = log_uniform
        lens = np.exp(rng.uniform(np.log(lo), np.log(hi + 1), n_sent)).astype(np.int64)
        lens = np.clip(lens, lo, hi)
    else:
        lens = np.clip(np.rint(rng.normal(mean_len, sd_len, n_sent)), min_len, max_len).astype(np.int64)
    total = int(lens.sum())
    n_surf = len(d.surf_off) - 1
    surf_len = np.diff(d.surf_off)
    mean_w = 2.2
    stream = np.empty(0, dtype=np.uint32)
    pieces = []
    have = 0
    while have < total:
        n_items = int((total - have) / mean_w * 1.15) + 64
        idx = _zipf_choice(rng, n_surf, n_items, 1.0)
        L = surf_len[idx]
        o = np.zeros(n_items + 1, dtype=np.int64)
        np.cumsum(L, out=o[1:])
        item_of = np.repeat(np.arange(n_items), L)
        src = d.surf_off[idx][item_of] + (np.arange(int(o[-1])) - o[:-1][item_of])
        chunk = d.surf_cps[src].copy()
        # replace a fraction of items by unknown-ish runs of the same length
        kind = rng.random(n_items)
        unk_item = kind < unk_frac
        sp_item = (kind >= unk_frac) & (kind < unk_frac + space_frac)
        flavour = rng.integers(0, 4, n_items)
        ch_unk = unk_item[item_of]
        fl = flavour[item_of]
        r = rng.integers(0, 1 << 30, len(chunk))
        rare = (0x4E00 + (r % (0x9FA5 - 0x4E00))).astype(np.uint32)
        chunk = np.where(ch_unk & (fl == 0), ASCII_ALPHA[r % len(ASCII_ALPHA)], chunk)
        chunk = np.where(ch_unk & (fl == 1), DIGITS[r % len(DIGITS)], chunk)
        chunk = np.where(ch_unk & (fl == 2), rare, chunk)
        chunk = np.where(ch_unk & (fl == 3), KATAKANA[r % len(KATAKANA)], chunk)
        chunk = np.where(sp_item[item_of], np.uint32(0x20), chunk)
        if astral_frac > 0:
            am = rng.random(len(chunk)) < astral_frac
            chunk = np.where(am, (0x1F300 + (r % 0x300)).astype(np.uint32), chunk)
        pieces.append(chunk.astype(np.uint32))
        have += len(chunk)
    stream = np.concatenate(pieces)[:total]
    if user_csv is not None and user_frac > 0:
        # splice user surfaces at the start of a fraction of sentences
        surfs = [ln.split(",")[0] for ln in user_csv.decode("utf-8").splitlines() if ln]
        starts = np.zeros(n_sent + 1, dtype=np.int64)
        np.cumsum(lens, out=starts[1:])
        pick = np.nonzero(rng.random(n_sent) < user_frac)[0]
        for si in pick.tolist():
            s = surfs[int(rng.integers(0, len(surfs)))]
            cp = np.array([ord(c) for c in s], dtype=np.uint32)
            room = int(lens[si])
            cp = cp[:room]
            p = int(starts[si]) + int(rng.integers(0, room - len(cp) + 1))
            stream[p:p + len(cp)] = cp
    utf8, bstart = encode_utf8(stream)
    cstart = np.zeros(n_sent + 1, dtype=np.int64)
    np.cumsum(lens, out=cstart[1:])
    offsets = bstart[cstart].astype(np.uint64)
    return utf8, offsets


def make_bigram_files(d, n_templates=6, vocab=24, pairs_per_template=260, seed=20260930):
    """bigram.right / bigram.left / bigram.cost (docs/small-dic.md of the reference) for the connection ids
    of `d`: every id gets one feature per template ("*" = no feature); costs exist for a random subset of
    (right feature, left feature) pairs, so a connection cost is the sum of the templates that hit."""
    rng = np.random.default_rng(seed)

    def feats(side, n_ids):
        rows = []
        for i in range(1, n_ids):
            cols = []
            for t in range(n_templates):
                r = rng.random()
                if r < 0.25:
                    cols.append("*")
                elif r < 0.30 and t == 2:
                    cols.append(f'"{side}{t}:a,b"')  # quoted field holding a comma (raw_connector.rs:418-445)
                else:
                    cols.append(f"{side}{t}:v{int(_zipf_choice(rng, vocab, 1, 0.7)[0])}")
            rows.append(f"{i}\t" + ",".join(cols[: n_templates - (i % 3 == 0)]))  # ragged rows: shorter get padded
        return "\n".join(rows) + "\n"

    right = feats("R", d.num_right)
    left = feats("L", d.num_left)
    lines = []
    for t in range(n_templates):
        seen = set()
        for _ in range(pairs_per_template):
            a, b = int(rng.integers(0, vocab)), int(rng.integers(0, vocab))
            if (a, b) in seen:
                continue
            seen.add((a, b))
            lines.append(f"R{t}:v{a}/L{t}:v{b}\t{int(rng.integers(-3000, 3000))}")
        if t == 2:
            lines.append(f"R{t}:a,b/L{t}:a,b\t-777")
            lines.append(f"R{t}:a,b/L{t}:v1\t555")
    lines.append("R0:v0/L0:v0\t42")  # a repeated pair: the later cost replaces the earlier one
    return right, left, "\n".join(lines) + "\n"


def make_mecab_model(num_left, num_right, n_templates=16, n_model_lines=20000, seed=20261015):
    """The files of a trained MeCab model shaped like unidic's (docs/small-dic.md of the reference): `feature.def`,
    `left-id.def` (ids 0..num_left-1), `right-id.def` (ids 0..num_right-1) and `model.def`, as a dict of str, for
    mecab::generate_bigram_info.  Every id gets a CSV feature row: one of 150 POS / conjugation tuples (six fields),
    then three lexical fields, often "*", sometimes a quoted field holding a comma, and some rows stop early.  The
    BIGRAM templates combine one to three fields, with `?` on the lexical ones; at most eight templates touch the
    lexical fields, so a Dual connector's matrix part stays POS-sized, as it does for unidic.  model.def has MeCab's
    header, UNIGRAM lines (skipped by the conversion), BOS/EOS sides, feature strings the ids never produce, and
    weights that truncate to a zero cost."""
    rng = np.random.default_rng(seed)
    pos1 = ["名詞", "動詞", "助詞", "形容詞", "副詞", "助動詞", "接尾辞", "補助記号", "代名詞", "連体詞", "接頭辞", "感動詞"]
    pos = []
    for k in range(150):
        p = [pos1[min(int(rng.geometric(0.3)) - 1, len(pos1) - 1)], f"細{int(rng.integers(0, 10))}",
             "*" if rng.random() < 0.5 else f"類{int(rng.integers(0, 8))}", "*" if rng.random() < 0.8 else "一般"]
        conj = rng.random() < 0.4
        p += [f"活用型{int(rng.integers(0, 24))}" if conj else "*", f"活用形{int(rng.integers(0, 12))}" if conj else "*"]
        pos.append(p)

    def rows(side, n_ids):
        out = ["0 BOS/EOS,*,*,*,*,*,*,*,*,*"]
        tup = _zipf_choice(rng, len(pos), n_ids, 1.1)
        lex = rng.integers(0, 4000, (n_ids, 3))
        star = rng.random((n_ids, 3)) < [0.3, 0.5, 0.7]
        quoted = rng.random(n_ids) < 0.03
        short = rng.random(n_ids) < 0.05
        for i in range(1, n_ids):
            f = list(pos[int(tup[i])]) + ["*" if star[i, j] else f"{side}語{int(lex[i, j])}" for j in range(3)]
            if quoted[i]:
                f[6] = f'"{f[6]},{int(lex[i, 0]) % 7}"'
            if short[i]:
                f = f[:7]
            out.append(f"{i} " + ",".join(f))
        return "\n".join(out) + "\n"

    templates = []  # (left template, right template)
    n_lex = min(8, max(1, n_templates // 3))
    for k in range(n_templates):
        if k < n_lex:
            idx = [int(rng.integers(0, 6)), 6 + k % 3]
        else:
            idx = sorted(set(rng.integers(0, 6, int(rng.integers(1, 4))).tolist()))
        if k == n_templates - 1:
            idx = idx + [10]  # past the end of every row: always "*"
        opt = [i >= 6 and i != 10 for i in idx]
        lt = f"B{k:02}:" + ",".join(f"%L{'?' if o else ''}[{i}]" for i, o in zip(idx, opt))
        rt = ",".join(f"%R{'?' if o else ''}[{i}]" for i, o in zip(idx, opt))
        templates.append((lt, rt))
    feature_def = "# synthetic feature.def\nUNIGRAM U00:%F[0]\nUNIGRAM U01:%F[0],%F?[1]\n\n" + "".join(
        f"BIGRAM {lt}/{rt}\n" for lt, rt in templates)
    left_id_def, right_id_def = rows("L", num_left), rows("R", num_right)

    def expansions(id_def, k, side):
        """The feature strings template k makes on one side (its map keys), for the model's weights to name."""
        tmpl = templates[k][side]
        out = set()
        for line in id_def.splitlines()[1:]:
            f = _split_csv(line.split(" ", 1)[1])
            s, ok, pos_ = [], True, 0
            while True:
                a = tmpl.find("%", pos_)
                if a < 0:
                    s.append(tmpl[pos_:])
                    break
                b = tmpl.index("]", a)
                i = int(tmpl[tmpl.index("[", a) + 1:b])
                v = f[i] if i < len(f) else "*"
                if tmpl[a + 2] == "?" and v == "*":
                    ok = False
                    break
                s.append(tmpl[pos_:a] + v)
                pos_ = b + 1
            if ok:
                out.add("".join(s))
        return sorted(out)

    # right-id.def names the left features (the left context's right ids), left-id.def the right ones
    lefts = [expansions(right_id_def, k, 0) for k in range(n_templates)]
    rights = [expansions(left_id_def, k, 1) for k in range(n_templates)]
    kind = rng.random(n_model_lines)
    tk = rng.integers(0, n_templates, n_model_lines)
    pick = rng.integers(0, 1 << 30, (n_model_lines, 2))
    w = rng.normal(0.0, 1.5, n_model_lines)
    w[rng.random(n_model_lines) < 0.02] = 1e-5  # |w| * 700 < 1: a zero cost
    lines = ["version: 102", "charset: UTF-8", "cost-factor: 700", "eval-size: 10", "unk-eval-size: 4", "bias: 0", ""]
    for n in range(n_model_lines):
        k, r = int(tk[n]), kind[n]
        ls, rs = lefts[k], rights[k]
        lf = ls[int(pick[n, 0]) % len(ls)] if ls else f"B{k:02}:"
        rf = rs[int(pick[n, 1]) % len(rs)] if rs else ""
        if r < 0.05:
            feat = f"U{k:02}:{rf}"  # a unigram feature: no '/' once BOS/EOS is gone
        elif r < 0.10:
            feat = f"BOS/EOS/{rf}"
        elif r < 0.15:
            feat = f"{lf}/BOS/EOS"
        elif r < 0.20:
            feat = f"{lf}/未知{int(pick[n, 1]) % 97}"
        else:
            feat = f"{lf}/{rf}"
        lines.append(f"{w[n]:.6f}\t{feat}")
    return {"feature.def": feature_def, "left-id.def": left_id_def, "right-id.def": right_id_def,
            "model.def": "\n".join(lines) + "\n"}


def _split_csv(row):
    """Fields of one CSV row with '"' quoting (the rows make_mecab_model writes)."""
    out, cur, q, i = [], [], False, 0
    while i < len(row):
        c = row[i]
        if q:
            if c == '"' and i + 1 < len(row) and row[i + 1] == '"':
                cur.append('"')
                i += 1
            elif c == '"':
                q = False
            else:
                cur.append(c)
        elif c == '"' and not cur:
            q = True
        elif c == ",":
            out.append("".join(cur))
            cur = []
        else:
            cur.append(c)
        i += 1
    out.append("".join(cur))
    return out
