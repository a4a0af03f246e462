"""Dictionaries and span lists that drive the required-token code (k_mark_spans, k_candidates_spans: span_postings,
count_span, span_match, csv_fields) to its limits (test data only).

* make_dictionary(): segment_fixtures.make_dictionary() with the features of the big lists rewritten into selector
  fields (ids, costs and rows unchanged), plus the crowded surface CROWD_SURFACE appended to both lexicons.  Record
  i of `k` / `l` / `m` (65 535 / 65 536 / 65 537 system homographs), of `n` (65 537 user homographs) and entry i of
  the 70 000 BIG (`X`) unk.def entries reads `<name>,<i % 2>,<i % 3>,<lo>,<best>`: lo = i < 65 535, best = the
  record big_best (the BIG entry BIG_UNK_BEST) picks.  SELECT names the patterns over those fields.
* the crowded surface: 40 user and 40 system homographs whose field 1 + k is 1 on a subset that splits the two
  lists into exactly CROWD_RUNS[k] runs of matching records together (pattern crowd_pattern(t)).
* make_quoted(): a small dictionary whose features quote fields (`"a,b"`, `""` escapes, empty and trailing fields,
  256 fields, multi-byte text); QUOTED_PATTERNS admits a known, distinct subset of the homographs of QUOTED_SURFACE
  or of the ALPHA unk.def entries.
* far_cases(), many_cases(), refused_cases(): sentences with spans of 32 766 ... 98 303 characters, 31 ... 200
  spans per sentence, and lists whose 33rd span is invalid."""
import segment_fixtures as sf

BIG_LISTS = {**sf.BIG_SYS, sf.BIG_USER[0]: sf.BIG_USER[1]}
# pattern name -> pattern over the selector fields `<name>,<i % 2>,<i % 3>,<lo>,<best>`
SELECT = {
    "all": None,
    "none": "NOPE",                # no record: the unknown fallback (every entry of the category)
    "best": "*,*,*,*,1",           # the big_best record only
    "lo": "*,*,*,1",               # the first 0xFFFF records: one full segment
    "hi": "*,*,*,0",               # the records from 65 535 on: a run that starts past u16
    "even": "*,0",                 # every second record: ~32 768 runs, the quadratic cand_at case
    "third": "*,*,0",              # every third record
}
CROWD_SURFACE = "WV"  # DEFAULT characters, in no other key
CROWD_N = 40
CROWD_RUNS = (3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33)


def selector(name, i, best):
    return f"{name},{i % 2},{i % 3},{int(i < sf.MAX_COUNT)},{int(i == best)}"


def crowd_split(t):
    """(user runs, system runs) of t runs: the user list takes the larger half."""
    return (t + 1) // 2, t // 2


def crowd_members(runs):
    """Records of a 40-homograph list in `runs` runs: single records at 0, 2, 4, ..., the last run reaching the
    list's end (so one run ends at the last record)."""
    if runs == 0:
        return set()
    out = {2 * r for r in range(runs - 1)}
    return out | set(range(2 * (runs - 1), CROWD_N))


def crowd_rows(lexicon):
    """The 40 rows of the crowded surface; lexicon 0 system, 1 user.  Costs differ so the best pick is unique."""
    rows = []
    for i in range(CROWD_N):
        bits = [int(i in crowd_members(crowd_split(t)[1 - lexicon])) for t in CROWD_RUNS]
        rows.append(f"{CROWD_SURFACE},{1 + i % 3},{1 + (i + lexicon) % 3},{100 + 7 * i + 3 * lexicon},"
                    f"wv{lexicon}.{i}," + ",".join(map(str, bits)))
    return rows


def crowd_pattern(t):
    return "*," * (1 + CROWD_RUNS.index(t)) + "1"


def _rewrite(csv, lists):
    """Features of the rows whose surface is in `lists` (name -> best record) -> selector fields."""
    out, seen = [], {}
    for line in csv.splitlines():
        head = line.split(",", 4)
        if head[0] in lists:
            i = seen.get(head[0], 0)
            seen[head[0]] = i + 1
            line = ",".join(head[:4] + [selector(head[0], i, lists[head[0]])])
        out.append(line)
    return "\n".join(out) + "\n"


def make_dictionary(seed=0):
    """(lex_csv, matrix, char_def, unk_def, user_csv, long_user_word): the segment fixtures' dictionary with selector
    features and the crowded surface."""
    lex, matrix, char_def, unk_def, user, long_word = sf.make_dictionary(seed)
    best = {s: sf.big_best(n) for s, n in BIG_LISTS.items()}
    lex = _rewrite(lex, {s: best[s] for s in sf.BIG_SYS}) + "\n".join(crowd_rows(0)) + "\n"
    user = _rewrite(user, {sf.BIG_USER[0]: best[sf.BIG_USER[0]]}) + "\n".join(crowd_rows(1)) + "\n"
    unk_def = _rewrite(unk_def, {"BIG": sf.BIG_UNK_BEST})
    return lex, matrix, char_def, unk_def, user, long_word


def select_expect(n, pattern, best):
    """The records of a selector list of n that `pattern` (a SELECT value) admits."""
    name = pattern and [k for k, v in SELECT.items() if v == pattern][0]
    keep = {None: lambda i: True, "none": lambda i: False, "best": lambda i: i == best,
            "lo": lambda i: i < sf.MAX_COUNT, "hi": lambda i: i >= sf.MAX_COUNT, "even": lambda i: i % 2 == 0,
            "third": lambda i: i % 3 == 0}[name]
    return [i for i in range(n) if keep(i)]


# One sentence per big source, the source spanned on its own character with each pattern; `b` next to it as in
# segment_fixtures.big_sentences.  (pattern name, sentence, span start byte)
BIG_SPAN_CASES = [(p, s, 0) for p in ("all", "none", "best", "lo", "hi") for s in ("kb", "lb", "mb", "nb", "Xb")] + \
                 [(p, "b" + c + "b", 1) for p in ("all", "best", "hi") for c in "lnX"]
QUADRATIC_CASES = [("even", "mb", 0), ("third", "nb", 0), ("even", "Xb", 0)]


def big_spans(cases):
    """(sentences, spans) of (pattern name, sentence, start) cases: the span covers the big character."""
    sents = [s for _, s, _ in cases]
    spans = [[(a, a + 1, SELECT[p])] for p, _, a in cases]
    return sents, spans


def crowd_cases():
    """(sentences, spans): the crowded surface spanned with every run count, at the start and after a word."""
    sents, spans = [], []
    for t in CROWD_RUNS:
        sents += [CROWD_SURFACE + "ab", "ab" + CROWD_SURFACE]
        spans += [[(0, 2, crowd_pattern(t))], [(2, 4, crowd_pattern(t))]]
    sents += [CROWD_SURFACE * 3]
    spans += [[(0, 2, crowd_pattern(33)), (2, 4, crowd_pattern(8)), (4, 6, crowd_pattern(9))]]
    return sents, spans


# --- quoted features ---------------------------------------------------------------------------------------------
QUOTED_SURFACE = "ab"
FIELDS_256 = ",".join(["f"] * 255 + ["w"])
QUOTED_FEATURES = [
    '"a,b",c',
    '"x""y",,z',
    '"",*,',
    FIELDS_256,
    ",".join(["f"] * 255 + ["v"]),
    '名詞,"固有,名詞",東京',
    ",".join(f"q{i}" for i in range(17)),
    ",".join(f"q{i}" for i in range(15)) + ",Q15,q16",
    '"a,b"',
    'a"b,"c""",d',
]
QUOTED_UNK = ['"a,b",unk', '"",*,', "記号,*,*"]
QUOTED_PATTERNS = {  # pattern -> the indices of QUOTED_FEATURES it admits
    '"a,b"': [0, 8],
    '"a,b",c': [0],
    '"x""y",,z': [1],
    '"*"': list(range(len(QUOTED_FEATURES))),  # a quoted star is still a wildcard
    '"",*,': [2],
    "*,*,": [2],                              # an empty field 2: the words with fewer fields lack it
    "*,,z": [1],
    ",".join(["*"] * 255 + ["w"]): [3],       # field index 255
    ",".join(["f"] * 16): [3, 4],             # 16 constrained fields
    ",".join(f"q{i}" for i in range(16)): [6],
    ",".join(f"q{i}" for i in range(15)) + ",*,q16": [6, 7],
    "*," * 16 + "q16": [6, 7],
    '名詞,"固有,名詞"': [5],
    '*,"固有,名詞",東京': [5],
    'a"b,c"': [9],                            # a quote inside an unquoted field is text
    '*,"c""",d': [9],
    '"a,b",unk': [],                          # no word: the unknown fallback
    "記号": [],
    "NOPE": [],
}
# the patterns that admit no word -> the ALPHA unk.def entries they admit (all of them when none matches)
QUOTED_UNK_PATTERNS = {'"a,b",unk': [0], "記号": [2], "NOPE": [0, 1, 2]}


def make_quoted():
    """(lex_csv, matrix, char_def, unk_def): QUOTED_SURFACE with QUOTED_FEATURES as its homographs, plus a few
    plain words; the ALPHA entries of unk.def with QUOTED_UNK."""
    lex = [f"{QUOTED_SURFACE},{1 + i % 2},{2 - i % 2},{10 * i - 40},{f}" for i, f in enumerate(QUOTED_FEATURES)]
    lex += ["a,1,1,200,名詞", "b,2,2,210,動詞", "abab,1,2,300,名詞"]
    matrix = "3 3\n" + "".join(f"{r} {l} {(r * 7 + l * 3) % 11 - 5}\n" for r in range(3) for l in range(3))
    char_def = "DEFAULT 0 1 0\nSPACE 0 1 0\nALPHA 1 1 3\n\n0x0020 SPACE\n0x0061..0x007A ALPHA\n"
    unk = ["DEFAULT,1,1,500,記号", "SPACE,0,0,50,空白"] + [f"ALPHA,{i},{2 - i},{300 + i},{f}"
                                                          for i, f in enumerate(QUOTED_UNK)]
    return "\n".join(lex) + "\n", matrix, char_def, "\n".join(unk) + "\n"


def quoted_cases():
    """(sentences, spans): QUOTED_SURFACE spanned with every pattern, alone, between words, and twice in a row."""
    sents, spans = [], []
    for p in QUOTED_PATTERNS:
        sents += ["ab", "abab" + "ab", "b ab a"]
        spans += [[(0, 2, p)], [(0, 2, p), (2, 4), (4, 6, p)], [(2, 4, p)]]
    return sents, spans


# --- far spans ----------------------------------------------------------------------------------------------------
FAR_LENGTHS = (32766, 32767, 32768, 65534, 65535, 98303)
PAD = 20


def far_cases(long_word):
    """(sentences, spans, ignore_space) of the far spans: over a `Z` run from 0, over an ALPHA run from its middle,
    behind SPACE_RUN with ignore_space, and over the long user word with a pattern that matches its feature and one
    that does not (the DEFAULT unknown word over 4 000 characters)."""
    sents, spans = [], []
    for n in FAR_LENGTHS:
        sents += ["Z" * n + "Zab", "z" * (n + 2 * PAD)]
        spans += [[(0, n)], [(PAD, PAD + n)]]
    lw = len(long_word)
    sents += [long_word + "ab", long_word + "ab"]
    spans += [[(0, lw, f"{long_word[:8]}0")], [(0, lw, "NOPE")]]
    isp_sents = [sf.SPACE_RUN + "z" * 40000 + "ab", sf.SPACE_RUN + long_word + "ab", sf.SPACE_RUN + long_word + "ab"]
    n = len(sf.SPACE_RUN)
    isp_spans = [[(n, n + 40000)], [(n, n + lw, f"{long_word[:8]}0")], [(n, n + lw, "NOPE")]]
    return sents, spans, isp_sents, isp_spans


# --- many spans ---------------------------------------------------------------------------------------------------
def _span_text(n_chars, seed):
    import numpy as np
    rng = np.random.default_rng([seed, 31])
    return "".join(rng.choice(list(sf.WORD_LETTERS + "cz"), n_chars))


def many_spans(text, count, first=0):
    """`count` spans from character `first` on: 1- and 2-character spans, adjacent in pairs, a one-character gap after
    every pair (all ASCII text, so characters are bytes)."""
    out, c = [], first
    while len(out) < count:
        out.append((c, c + 1))
        if len(out) < count:
            out.append((c + 1, c + 3))
        c += 4
    assert c <= len(text) + 1
    return out


def chunk_edge_spans():
    """Spans that end at the interior chunk edges 31 / 32 / 33 and 63 / 64 / 65, and one over 32 .. 96."""
    return [(0, 31), (31, 32), (32, 33), (34, 63), (63, 64), (64, 65), (65, 97), (97, 98)]


MANY_COUNTS = (31, 32, 33, 64, 65, 200)


def many_cases():
    """(sentences, spans): 31 ... 200 spans per sentence, the chunk-edge spans, a span over a 150 000-character
    sentence, and one with 65 spans on a text with multi-byte characters."""
    sents, spans = [], []
    for k, count in enumerate(MANY_COUNTS):
        t = _span_text(4 * count + 8, k)
        sents.append(t)
        spans.append(many_spans(t, count, first=k % 3))
    t = _span_text(130, 9)
    sents.append(t)
    spans.append(chunk_edge_spans())
    sents.append("Z" * sf.RUN_LEN)
    spans.append([(0, sf.RUN_LEN)])
    mb = "".join("ab東" for _ in range(80))  # 5 bytes per 3 characters
    sents.append(mb)
    spans.append([(5 * i, 5 * i + 2) for i in range(65)])
    return sents, spans


def refused_cases():
    """Lists (for a batch of one sentence) whose 33rd span is invalid: it overlaps the 32nd; an explicit boundary
    falls inside it at a chunk edge; it ends off a UTF-8 lead byte.  (sentence, spans, boundaries)"""
    t = _span_text(400, 3)
    good = many_spans(t, 32)
    mb = "ab東" * 120
    good_mb = [(5 * i, 5 * i + 2) for i in range(32)]
    return [
        (t, good + [(good[-1][1] - 1, good[-1][1] + 3)], []),
        (t, good + [(good[-1][1] + 1, good[-1][1] + 300)], [192]),  # character 192: a chunk edge inside the span
        (mb, good_mb + [(5 * 32, 5 * 32 + 3)], []),                 # byte 163 is inside 東 (bytes 162..164)
    ]
